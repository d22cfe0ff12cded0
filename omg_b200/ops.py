"""Host-side launchers: torch tensors (device memory + stream plumbing only) -> C-ABI descriptors.

All activations are channels-last fp16: (B, H, W, C), equivalently (B, H*W tokens, C).  `linear`, `conv3x3`,
`upsample2x_conv3x3`, `groupnorm` and `softmax_rows` also run in bf16 (the VAE decoder's path): the storage type comes
from the tensors, outputs are allocated in it, and mixing fp16 and bf16 operands raises ValueError.
"""
import ctypes as C

import torch

from . import _lib as L


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


_DTYPE_NAMES = {torch.float16: "fp16", torch.bfloat16: "bf16"}


def _chk(t: torch.Tensor, dtype):
    if not t.is_cuda or t.dtype != dtype:
        raise ValueError(f"expected a CUDA {_DTYPE_NAMES[dtype]} tensor (there is no CPU path)")


def _chk16(t: torch.Tensor):
    _chk(t, torch.float16)


def _op_dtype(x: torch.Tensor, *others):
    """Storage type of an op that runs in fp16 or bf16: that of x.  A bf16 op takes only bf16 operands; an fp16 op
    rejects bf16 ones (None entries are skipped)."""
    if not x.is_cuda or x.dtype not in _DTYPE_NAMES:
        raise ValueError("expected a CUDA fp16 or bf16 tensor (there is no CPU path)")
    for t in others:
        if t is None:
            continue
        if torch.bfloat16 in (x.dtype, t.dtype) and t.dtype != x.dtype:
            raise ValueError(f"mixed operand types: {x.dtype} and {t.dtype} (fp16 and bf16 do not mix)")
    return x.dtype


def view4(t: torch.Tensor, dtype=torch.float16) -> L.View4:
    """(B,H,W,C) tensor (any pixel strides, unit channel stride) or 2-D [M,K] matrix -> omg_view4."""
    _chk(t, dtype)
    if t.dim() == 2:
        assert t.stride(1) == 1
        return L.View4(t.data_ptr(), t.shape[1], t.shape[0], 1, 1, t.stride(0), t.stride(0) * t.shape[0],
                       t.stride(0) * t.shape[0])
    assert t.dim() == 4 and t.stride(3) == 1
    B, H, W, Cc = t.shape
    return L.View4(t.data_ptr(), Cc, W, H, B, t.stride(2), t.stride(1), t.stride(0))


def _ptr(t):
    return None if t is None else t.data_ptr()


class LaunchPlan:
    """omg_plan (include/omg_b200.h): the launches of one forward recorded at the C ABI and replayed from C with no
    descriptor building - what a non-Python host holds instead of the reference's `self.unet(...)` call
    (src/pipelines/lora_pipeline.py:558-567).  Everything a recorded launch points to must outlive the plan (the
    executor's persistent workspace does; tensors allocated inside the recorded region do not)."""

    def __init__(self):
        self._lib = L.load()
        self._h = self._lib.omg_plan_create()
        if not self._h:
            raise RuntimeError("omg_plan_create failed")

    def __enter__(self):
        L.check(self._lib.omg_plan_record_begin(self._h), "omg_plan_record_begin")
        return self

    def __exit__(self, *exc):
        L.check(self._lib.omg_plan_record_end(self._h), "omg_plan_record_end")
        return False

    def __len__(self):
        return int(self._lib.omg_plan_length(self._h))

    def clear(self):
        L.check(self._lib.omg_plan_clear(self._h), "omg_plan_clear")

    def run(self, stream=None):
        L.check(self._lib.omg_plan_run(self._h, _stream() if stream is None else stream), "omg_plan_run")

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.omg_plan_destroy(h)


def gemm(a_views, segs, w, N, Ktot, d_view, bias=None, rowvec=None, rowvec_ld=0, residual=None, residual_ld=0,
         epilogue=L.EPI_NONE, block_n=0, w2=None, stats_out=None, ln=None, cta_pair=0, row_groups=None, colstats=None,
         residual_f32=None, out_f32=None):
    d = L.GemmDesc()
    d.dtype = L.DTYPE_BF16 if w.dtype == torch.bfloat16 else L.DTYPE_F16  # of every 16-bit operand (checked by the ops)
    if residual_f32 is not None:   # [pixels, N] fp32 twins of the residual trunk (see omg_gemm_desc)
        d.residual_f32, d.residual_f32_ld = residual_f32.data_ptr(), residual_f32.stride(-2)
    if out_f32 is not None:
        d.out_f32, d.out_f32_ld = out_f32.data_ptr(), out_f32.stride(-2)
    d.cta_pair = cta_pair
    if colstats is not None:  # (partials [B, rb_total, N, 2] fp32, first block this launch fills)
        part, rb0 = colstats
        d.col_stats_out, d.col_stats_rb0, d.col_stats_rb_total = part.data_ptr(), rb0, part.shape[1]
    if row_groups is not None:  # per-stream weight planes: w is [len(row_groups) * N, Ktot]
        d.w_group_planes = d.n_col_groups = len(row_groups)
        for i, e in enumerate(row_groups):
            d.col_group_end[i] = e
    d.n_a = len(a_views)
    for i, v in enumerate(a_views):
        d.a[i] = v
    d.n_segs = len(segs)
    for i, s in enumerate(segs):
        d.segs[i] = L.Seg(*s) if len(s) == 7 else L.Seg(*s, 0)
    d.w = w.data_ptr()
    d.N, d.Ktot = N, Ktot
    if w2 is not None:
        d.w2, d.K2tot = w2.data_ptr(), w2.shape[1]
    d.d = d_view
    d.bias = _ptr(bias)
    d.rowvec = _ptr(rowvec)
    d.rowvec_ld = rowvec_ld
    d.residual = _ptr(residual)
    d.residual_ld = residual_ld
    d.epilogue = epilogue
    d.block_n = block_n
    if stats_out is not None:
        d.row_stats_out = stats_out.data_ptr()
    if ln is not None:  # folded LayerNorm: (stats [parts, rows, 2] fp32, parts, rows per part, row offset, dim, eps, c1, c2)
        stats, parts, stride, row0, dim, eps, c1, c2, group_ends = ln
        d.row_stats_in = stats.data_ptr() + row0 * 8
        d.row_stats_parts, d.row_stats_stride, d.ln_dim, d.ln_eps = parts, stride, dim, eps
        d.col_c1, d.col_c2 = c1.data_ptr(), c2.data_ptr()
        d.n_col_groups = len(group_ends)
        for i, e in enumerate(group_ends):
            d.col_group_end[i] = e
    L.check(L.load().omg_gemm(C.byref(d), _stream()), "omg_gemm")


def gemm_plan(N, epilogue, W, H=1, B=1):
    """(block_n, n_tiles) omg_gemm will use; n_tiles = number of row-statistics partials a producer emits."""
    bn, nt = C.c_int(0), C.c_int(0)
    L.check(L.load().omg_gemm_plan(N, epilogue, W, H, B, C.byref(bn), C.byref(nt)), "omg_gemm_plan")
    return bn.value, nt.value


def colstats_blocks(W, H=1):
    """32-pixel column-statistics blocks one omg_gemm launch over an output grid (W, H) writes per image."""
    return L.load().omg_gemm_colstats_blocks(W, H)


def linear(x, w, bias=None, residual=None, out=None, epilogue=L.EPI_NONE, extra=None, block_n=0, lora=None,
           stats_out=None, ln=None, cta_pair=0, row_groups=None, colstats=None, residual_f32=None, out_f32=None):
    """out[M, N'] = epi(x[M,K] @ w[N, :K]^T (+ extra K-segments) + bias) + residual.

    `extra` = list of (tensor [M,Ki], column offset into w): further K-segments of the same weight matrix.
    `lora`  = (t [M,R], w2 [N,R]): un-merged LoRA delta  t @ w2^T  with t = A x (scales folded into w2).
    fp16 or bf16 (x's type; bf16 without epilogue, LoRA, statistics, LayerNorm fold, row groups or fp32 twins).
    """
    dt = _op_dtype(x, w, bias, residual, out, *[t for t, _ in (extra or [])], *(lora or ()))
    M, K = x.shape
    N, Ktot = w.shape
    if row_groups is not None:
        N //= len(row_groups)
    n_out = N // 2 if epilogue == L.EPI_GEGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=dt, device=x.device)
    views = [view4(x, dt)]
    segs = [(0, 0, 0, 0, K, 0)]
    for t, off in (extra or []):
        views.append(view4(t, dt))
        segs.append((len(views) - 1, 0, 0, 0, t.shape[1], off))
    w2 = None
    if lora is not None:
        t, w2 = lora
        views.append(view4(t, dt))
        segs.append((len(views) - 1, 0, 0, 0, t.shape[1], 0, 1))
    # colstats: partials [B, rb, N, 2] of an output of B images x HW tokens; the [M, N] GEMM sees them as one image
    # of M rows, which is the same memory when no 128-row tile straddles two images (HW % 128 == 0, caller's duty)
    cs = None if colstats is None else (colstats.view(1, -1, colstats.shape[2], 2), 0)
    gemm(views, segs, w, N, Ktot, view4(out, dt), bias=bias, residual=residual,
         residual_ld=0 if residual is None else residual.stride(0), epilogue=epilogue, block_n=block_n, w2=w2,
         stats_out=stats_out, ln=ln, cta_pair=cta_pair, row_groups=row_groups, colstats=cs,
         residual_f32=residual_f32, out_f32=out_f32)
    return out


def _taps3x3(Cin, a_idx=0, c0=0, k0=0):
    return [(a_idx, kx - 1, ky - 1, c0, Cin, k0 + (ky * 3 + kx) * Cin) for ky in range(3) for kx in range(3)]


def _image_groups(row_groups, pixels):
    """Cumulative image counts of the streams -> group ends in pixels of a launch's output grid (omg_gemm_desc
    col_group_end: on a spatial grid every boundary is a whole number of images)."""
    return None if row_groups is None else [e * pixels for e in row_groups]


def conv3x3(x, w, bias=None, rowvec=None, residual=None, out=None, shortcut=None, block_n=0, cta_pair=0, colstats=None,
            residual_f32=None, out_f32=None, row_groups=None):
    """3x3 / stride 1 / pad 1 conv over (B,H,W,Cin).  w = [N, 9*Cin (+ shortcut K)] packed (ky, kx, c).

    row_groups = cumulative image counts [n_1, n_1 + n_2, ..., B] of streams with weights of their own (per-stream LoRA
    merged into the conv): w is then the stack [len(row_groups) * N, K] and images [n_(g-1), n_g) use plane g.  The same
    argument of conv3x3_s2 and upsample2x_conv3x3 counts images too; each launch converts it to pixels of ITS output
    grid (H/2 x W/2 there, the H x W phase grid of the four up-sampler launches).

    shortcut = list of (tensor (B,H,W,Ci), weight column offset): 1x1-conv K-segments added to the same accumulator
    (ResnetBlock2D conv_shortcut).  rowvec [B, N] is added per image (time-embedding projection).
    fp16 or bf16 (x's type; bf16 with bias, residual and shortcut only).
    """
    dt = _op_dtype(x, w, bias, rowvec, residual, out, *[t for t, _ in (shortcut or [])])
    B, H, W, Cin = x.shape
    N, Ktot = w.shape
    if row_groups is not None:
        N //= len(row_groups)
    if out is None:
        out = torch.empty((B, H, W, N), dtype=dt, device=x.device)
    views = [view4(x, dt)]
    segs = _taps3x3(Cin)
    for t, off in (shortcut or []):
        views.append(view4(t, dt))
        segs.append((len(views) - 1, 0, 0, 0, t.shape[3], off))
    gemm(views, segs, w, N, Ktot, view4(out, dt), bias=bias, rowvec=rowvec,
         rowvec_ld=0 if rowvec is None else rowvec.stride(0),
         residual=residual, residual_ld=0 if residual is None else N, block_n=block_n, cta_pair=cta_pair,
         colstats=None if colstats is None else (colstats, 0), residual_f32=residual_f32, out_f32=out_f32,
         row_groups=_image_groups(row_groups, H * W))
    return out


def conv3x3_s2(x, w, bias=None, out=None, block_n=0, colstats=None, row_groups=None, epilogue=L.EPI_NONE):
    """3x3 / stride 2 / pad 1 conv (Downsample2D): A operands are the four stride-2 phase views of x.
    row_groups: per-stream weight planes, see conv3x3.  epilogue: activation applied after the bias (the tanh-GELU of the
    SAM encoder's stride-2 convs)."""
    B, H, W, Cin = x.shape
    N, Ktot = w.shape
    if row_groups is not None:
        N //= len(row_groups)
    assert H % 2 == 0 and W % 2 == 0
    if out is None:
        out = torch.empty((B, H // 2, W // 2, N), dtype=torch.float16, device=x.device)
    views = [view4(x[:, py::2, px::2, :]) for py in range(2) for px in range(2)]
    segs = []
    for ky in range(3):
        for kx in range(3):
            py, oy = (1, -1) if ky == 0 else ((0, 0) if ky == 1 else (1, 0))
            px, ox = (1, -1) if kx == 0 else ((0, 0) if kx == 1 else (1, 0))
            segs.append((py * 2 + px, ox, oy, 0, Cin, (ky * 3 + kx) * Cin))
    gemm(views, segs, w, N, Ktot, view4(out), bias=bias, epilogue=epilogue, block_n=block_n,
         colstats=None if colstats is None else (colstats, 0), row_groups=_image_groups(row_groups, (H // 2) * (W // 2)))
    return out


def upsample2x_conv3x3(x, w, bias=None, out=None, block_n=0, colstats=None, row_groups=None):
    """nearest-2x upsample followed by 3x3 conv (Upsample2D) without materialising the upsampled tensor:
    each output phase (py,px) is a 9-tap conv over x with shifted taps, stored through a strided output view.
    fp16 or bf16 (x's type; bf16 without column statistics).  row_groups: per-stream weight planes, see conv3x3."""
    dt = _op_dtype(x, w, bias, out)
    B, H, W, Cin = x.shape
    N, Ktot = w.shape
    if row_groups is not None:
        N //= len(row_groups)
    if out is None:
        out = torch.empty((B, 2 * H, 2 * W, N), dtype=dt, device=x.device)
    xv = view4(x, dt)
    off = {0: (-1, 0, 0), 1: (0, 0, 1)}
    for py in range(2):
        for px in range(2):
            segs = [(0, off[px][kx], off[py][ky], 0, Cin, (ky * 3 + kx) * Cin) for ky in range(3) for kx in range(3)]
            cs = None if colstats is None else (colstats, (py * 2 + px) * colstats_blocks(W, H))
            gemm([xv], segs, w, N, Ktot, view4(out[:, py::2, px::2, :], dt), bias=bias, block_n=block_n, colstats=cs,
                 row_groups=_image_groups(row_groups, H * W))
    return out


def attention(q, k, v, out, heads, n_q, n_kv, items, q_col0=0, k_col0=0, v_col0=0, out_col0=0, scale=0.125,
              out_weight=1.0, accumulate=False, causal=False):
    """q/k/v/out: [batch, tokens, ld] fp16.  items: list of (out_b, q_b, k_b, v_b)."""
    for t in (q, k, v, out):
        _chk16(t)
        assert t.dim() == 3 and t.stride(2) == 1
    d = L.AttnDesc()
    d.q, d.q_ld, d.q_bs, d.q_col0 = q.data_ptr(), q.stride(1), q.stride(0), q_col0
    d.k, d.k_ld, d.k_bs, d.k_col0 = k.data_ptr(), k.stride(1), k.stride(0), k_col0
    d.v, d.v_ld, d.v_bs, d.v_col0 = v.data_ptr(), v.stride(1), v.stride(0), v_col0
    d.out, d.out_ld, d.out_bs, d.out_col0 = out.data_ptr(), out.stride(1), out.stride(0), out_col0
    d.n_q, d.n_kv, d.heads, d.head_dim = n_q, n_kv, heads, 64
    d.n_items = len(items)
    for i, (ob, qb, kb, vb) in enumerate(items):
        d.out_b[i], d.q_b[i], d.k_b[i], d.v_b[i] = ob, qb, kb, vb
    d.scale, d.out_weight, d.accumulate, d.causal = scale, out_weight, int(accumulate), int(causal)
    L.check(L.load().omg_attention(C.byref(d), _stream()), "omg_attention")
    return out


def attention_small_ws(n_items, heads, n_q, n_kv, device="cuda"):
    """fp32 workspace of the split-key path of attention_small (OMG_ATTN_SMALL_WS_FLOATS)."""
    n = min(n_items, L.OMG_ATTN_MAX_ITEMS) * heads * n_q * ((n_kv + 127) // 128) * 36
    return torch.empty(n, dtype=torch.float32, device=device)


def attention_small(q, k, v, out, heads, head_dim, n_q, n_kv, q_col0=0, k_col0=0, v_col0=0, out_col0=0, scale=None,
                    ws=None, items=None):
    """softmax(scale Q K^T) V per head for head_dim 16 | 32 with one short side (<= 64 tokens): q/k/v/out are
    [batch, tokens, ld] fp16 column views (a head's columns at col0 + head_dim * h).  items: list of (out_b, q_b, k_b, v_b),
    default one per batch; more than 16 items are issued as several launches.  ws: attention_small_ws(...) when
    n_kv > 64 (the split-key path)."""
    for t in (q, k, v, out):
        _chk16(t)
        assert t.dim() == 3 and t.stride(2) == 1
    if items is None:
        items = [(b, b, b, b) for b in range(out.shape[0])]
    if n_kv > 64 and ws is None:
        ws = attention_small_ws(len(items), heads, n_q, n_kv, q.device)
    for i0 in range(0, len(items), L.OMG_ATTN_MAX_ITEMS):
        chunk = items[i0:i0 + L.OMG_ATTN_MAX_ITEMS]
        d = L.AttnDesc()
        d.q, d.q_ld, d.q_bs, d.q_col0 = q.data_ptr(), q.stride(1), q.stride(0), q_col0
        d.k, d.k_ld, d.k_bs, d.k_col0 = k.data_ptr(), k.stride(1), k.stride(0), k_col0
        d.v, d.v_ld, d.v_bs, d.v_col0 = v.data_ptr(), v.stride(1), v.stride(0), v_col0
        d.out, d.out_ld, d.out_bs, d.out_col0 = out.data_ptr(), out.stride(1), out.stride(0), out_col0
        d.n_q, d.n_kv, d.heads, d.head_dim = n_q, n_kv, heads, head_dim
        d.n_items = len(chunk)
        for i, (ob, qb, kb, vb) in enumerate(chunk):
            d.out_b[i], d.q_b[i], d.k_b[i], d.v_b[i] = ob, qb, kb, vb
        d.scale = head_dim ** -0.5 if scale is None else scale
        d.out_weight, d.accumulate, d.causal = 1.0, 0, 0
        L.check(L.load().omg_attention_small(C.byref(d), _ptr(ws), _stream()), "omg_attention_small")
    return out


def attention_relpos(qkv, H, W, heads, head_dim, rel_pos_h, rel_pos_w, window=0, k_bias=None, v_bias=None, out=None,
                     q_col0=None, k_col0=None, v_col0=None, out_col0=0, scale=None):
    """SAM ViT attention with decomposed relative-position bias (omg_attention_relpos).  qkv: fp16 [B, H*W, ld] in token
    order, q / k / v of head h at columns q_col0 / k_col0 / v_col0 + head_dim * h (default 0, C, 2C: the qkv Linear's
    output).  rel_pos_h / rel_pos_w: fp16 [2S - 1, head_dim] (S = window, or H / W when window = 0).  k_bias / v_bias:
    fp16 [C], the qkv bias of k and v - the padded tokens' key and value when H or W is not a multiple of the window.
    Returns out, fp16 [B, H*W, >= C] (allocated [B, H*W, C] when None)."""
    Cd = heads * head_dim
    q_col0 = 0 if q_col0 is None else q_col0
    k_col0 = Cd if k_col0 is None else k_col0
    v_col0 = 2 * Cd if v_col0 is None else v_col0
    for t in (qkv, rel_pos_h, rel_pos_w, k_bias, v_bias, out):
        if t is not None:
            _chk16(t)
    assert qkv.dim() == 3 and qkv.stride(2) == 1 and qkv.shape[1] == H * W
    for t in (rel_pos_h, rel_pos_w, k_bias, v_bias):
        assert t is None or t.is_contiguous()
    if out is None:
        out = torch.empty(qkv.shape[0], H * W, Cd, dtype=torch.float16, device=qkv.device)
    assert out.dim() == 3 and out.stride(2) == 1
    d = L.AttnRelposDesc()
    d.qkv, d.ld, d.bs, d.q_col0, d.k_col0, d.v_col0 = qkv.data_ptr(), qkv.stride(1), qkv.stride(0), q_col0, k_col0, v_col0
    d.out, d.out_ld, d.out_bs, d.out_col0 = out.data_ptr(), out.stride(1), out.stride(0), out_col0
    d.B, d.H, d.W, d.heads, d.head_dim, d.window = qkv.shape[0], H, W, heads, head_dim, window
    d.rel_pos_h, d.rel_h_len = rel_pos_h.data_ptr(), rel_pos_h.shape[0]
    d.rel_pos_w, d.rel_w_len = rel_pos_w.data_ptr(), rel_pos_w.shape[0]
    d.k_bias, d.v_bias = _ptr(k_bias), _ptr(v_bias)
    d.scale = head_dim ** -0.5 if scale is None else scale
    L.check(L.load().omg_attention_relpos(C.byref(d), _stream()), "omg_attention_relpos")
    return out


def sam_mask_head(up1, ln_w, ln_b, w2, b2, hyper, M, eps=1e-6, out=None):
    """SAM output_upscaling after ConvTranspose2d #1 + hypernetwork product (omg_sam_mask_head).  up1 fp16
    [B, 64, 64, 2, 2, 64] (or [B*4096, 256]); w2 fp32 [2, 2, 64, 32]; hyper fp16 (B, M, 32) view with unit channel
    stride -> fp32 (B, M, 256, 256) low-res logits."""
    _chk16(up1)
    _chk16(hyper)
    assert up1.is_contiguous() and hyper.stride(-1) == 1
    B = up1.numel() // (4096 * 256)
    if out is None:
        out = torch.empty((B, M, 256, 256), dtype=torch.float32, device=up1.device)
    L.check(L.load().omg_sam_mask_head(up1.data_ptr(), ln_w.data_ptr(), ln_b.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                                       hyper.data_ptr(), hyper.stride(0), hyper.stride(1), B, M, float(eps), out.data_ptr(),
                                       _stream()), "omg_sam_mask_head")
    return out


def sam_postprocess(lowres, input_size, original_size, mid=1024, threshold=0.0, mask=None, logits=None,
                    return_mask=True, return_logits=False):
    """postprocess_masks + threshold (omg_sam_postprocess): lowres fp32 (B, M, low, low) -> (bool mask, fp32 logits)
    at original_size (either None when not requested)."""
    assert lowres.is_cuda and lowres.dtype == torch.float32 and lowres.is_contiguous()
    B, M, low, _ = lowres.shape
    H, W = original_size
    if return_mask and mask is None:
        mask = torch.empty((B, M, H, W), dtype=torch.bool, device=lowres.device)
    if return_logits and logits is None:
        logits = torch.empty((B, M, H, W), dtype=torch.float32, device=lowres.device)
    L.check(L.load().omg_sam_postprocess(lowres.data_ptr(), B * M, low, mid, int(input_size[0]), int(input_size[1]), H, W,
                                         float(threshold), _ptr(mask), _ptr(logits), _stream()), "omg_sam_postprocess")
    return mask, logits


def groupnorm(x1, gamma, beta, eps, silu, x2=None, out=None, stats_ws=None):
    """GroupNorm(32)(cat([x1, x2], channel)) [+ SiLU]; x: (B, H, W, C) or (B, HW, C).  fp16 or bf16 (x1's type, also
    that of x2, gamma, beta and out); fp32 statistics either way."""
    dt = _op_dtype(x1, x2, gamma, beta, out)
    B = x1.shape[0]
    C1 = x1.shape[-1]
    HW = x1.numel() // (B * C1)
    C2 = 0 if x2 is None else x2.shape[-1]
    assert x1.is_contiguous() and (x2 is None or x2.is_contiguous())
    if out is None:
        out = torch.empty((*x1.shape[:-1], C1 + C2), dtype=dt, device=x1.device)
    if stats_ws is None:
        stats_ws = torch.empty(B * (10240 + 64 * 256), dtype=torch.float32, device=x1.device)
    name = "omg_groupnorm_bf16" if dt == torch.bfloat16 else "omg_groupnorm"
    L.check(getattr(L.load(), name)(x1.data_ptr(), C1, _ptr(x2), C2, B, HW, gamma.data_ptr(), beta.data_ptr(),
                                    float(eps), int(silu), stats_ws.data_ptr(), out.data_ptr(), _stream()), name)
    return out


def colstats(x, out=None):
    """Per-channel (sum, sumsq) partials of a stored (B, HW.., C) tensor, one per 32-row block: [B, ceil(HW/32), C, 2]."""
    _chk16(x)
    assert x.is_contiguous()
    B, Cc = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * Cc)
    if out is None:
        out = torch.empty((B, (HW + 31) // 32, Cc, 2), dtype=torch.float32, device=x.device)
    assert out.shape[0] >= B and out.shape[1] == (HW + 31) // 32 and out.shape[2] == Cc
    L.check(L.load().omg_colstats(x.data_ptr(), Cc, B, HW, out.data_ptr(), _stream()), "omg_colstats")
    return out


def groupnorm_apply(x1, part1, gamma, beta, eps, silu, x2=None, part2=None, out=None, stats_ws=None):
    """GroupNorm(32)(cat([x1, x2], channel)) [+ SiLU] with the statistics taken from per-channel partials
    (omg_gemm colstats / ops.colstats): no statistics pass over x."""
    _chk16(x1)
    B, C1 = x1.shape[0], x1.shape[-1]
    HW = x1.numel() // (B * C1)
    C2 = 0 if x2 is None else x2.shape[-1]
    assert x1.is_contiguous() and (x2 is None or x2.is_contiguous())
    assert part1.shape[0] == B and part1.shape[2] == C1 and (x2 is None or (part2.shape[0] == B and part2.shape[2] == C2))
    if out is None:
        out = torch.empty((*x1.shape[:-1], C1 + C2), dtype=torch.float16, device=x1.device)
    if stats_ws is None:
        stats_ws = torch.empty(B * (10240 + 64 * 256), dtype=torch.float32, device=x1.device)
    L.check(L.load().omg_groupnorm_apply(x1.data_ptr(), C1, part1.data_ptr(), part1.shape[1], _ptr(x2), C2, _ptr(part2),
                                         0 if part2 is None else part2.shape[1], B, HW, gamma.data_ptr(), beta.data_ptr(),
                                         float(eps), int(silu), stats_ws.data_ptr(), out.data_ptr(), _stream()),
            "omg_groupnorm_apply")
    return out


def dwconv(x, w, bias=None, out=None, ksize=3, stride=1, act=0):
    """Depthwise k x k conv ("same" padding) over (B, H, W, C) rows that may be strided views along the channel axis
    (x.stride(2) = row stride); w tap-major [k*k, C]; act 1 = tanh-GELU."""
    _chk16(x)
    B, H, W, Cc = x.shape
    assert x.stride(3) == 1 and x.stride(1) == x.stride(2) * W and x.stride(0) == x.stride(1) * H
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    if out is None:
        out = torch.empty((B, Ho, Wo, Cc), dtype=torch.float16, device=x.device)
    assert out.stride(3) == 1 and out.stride(1) == out.stride(2) * Wo and out.stride(0) == out.stride(1) * Ho
    L.check(L.load().omg_dwconv(x.data_ptr(), w.data_ptr(), _ptr(bias), out.data_ptr(), B, H, W, Cc, x.stride(2), out.stride(2),
                                ksize, stride, int(act), _stream()), "omg_dwconv")
    return out


def group1x1(x, w, out):
    """Grouped 1x1 conv, square groups of 32 channels: x (.., C) rows strided, w [C, 32], out (.., C) rows strided."""
    _chk16(x)
    Cc = x.shape[-1]
    pixels = x.numel() // Cc
    L.check(L.load().omg_group1x1(x.data_ptr(), w.data_ptr(), out.data_ptr(), pixels, Cc, x.stride(-2), out.stride(-2), 32, _stream()),
            "omg_group1x1")
    return out


def relu_linear_attention(qkv, heads, dim=32, eps=1e-15, out=None):
    """LiteMLA core: qkv (B, N, heads*3*dim) contiguous -> (B, N, heads*dim)."""
    _chk16(qkv)
    assert qkv.is_contiguous()
    B, N, _ = qkv.shape
    if out is None:
        out = torch.empty((B, N, heads * dim), dtype=torch.float16, device=qkv.device)
    L.check(L.load().omg_relu_linear_attention(qkv.data_ptr(), out.data_ptr(), B, N, heads, dim, float(eps), _stream()),
            "omg_relu_linear_attention")
    return out


def resize_bicubic(x, Ho, Wo, out=None):
    """F.interpolate(mode='bicubic', align_corners=False) over (B, H, W, C)."""
    _chk16(x)
    assert x.is_contiguous()
    B, H, W, Cc = x.shape
    if out is None:
        out = torch.empty((B, Ho, Wo, Cc), dtype=torch.float16, device=x.device)
    L.check(L.load().omg_resize_bicubic(x.data_ptr(), out.data_ptr(), B, H, W, Cc, Ho, Wo, _stream()), "omg_resize_bicubic")
    return out


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    _chk16(x)
    assert x.is_contiguous()
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    if out is None:
        out = torch.empty_like(x)
    L.check(L.load().omg_layernorm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), rows, Cc,
                                   float(eps), _stream()), "omg_layernorm")
    return out


def _fuse_desc(d, noise_main, noise_concepts, masks, guidance, sigma, sigma_next, latents, next_main_in,
               next_concept_in, latents_f16):
    d.noise_main = noise_main.data_ptr()
    d.n_concepts = len(noise_concepts)
    for i, (n, m) in enumerate(zip(noise_concepts, masks)):
        d.noise_concept[i] = _ptr(n)
        d.mask[i] = _ptr(m)
    d.guidance, d.sigma, d.sigma_next = float(guidance), float(sigma), float(sigma_next)
    d.latents = latents.data_ptr()
    d.next_main_in = _ptr(next_main_in)
    d.next_concept_in = _ptr(next_concept_in)
    d.latents_f16 = _ptr(latents_f16)
    d.HW = latents.shape[1] * latents.shape[2] if latents.dim() == 4 else latents.shape[1]


def fuse_step(noise_main, noise_concepts, masks, guidance, sigma, sigma_next, latents, next_main_in=None,
              next_concept_in=None, latents_f16=None):
    d = L.FuseDesc()
    _fuse_desc(d, noise_main, noise_concepts, masks, guidance, sigma, sigma_next, latents, next_main_in,
               next_concept_in, latents_f16)
    L.check(L.load().omg_fuse_step(C.byref(d), _stream()), "omg_fuse_step")


def solver_step(noise_main, noise_concepts, masks, guidance, coeffs, latents, next_main_in=None, next_concept_in=None,
                latents_f16=None, history=None, store_x0=False, noise=None):
    """omg_fuse_step's fusion and guidance with the update of `coeffs` (omg_b200.scheduler.StepCoeffs):
    x0 = c_x x + c_eps eps, x' = a x + b x0 + c history + d noise, next inputs = x' * s.  history: fp32 (2, h, w, 4),
    overwritten with x0 when store_x0; noise: fp16 (2, 4, h, w) as torch.randn draws it."""
    d = L.SolverDesc()
    _fuse_desc(d.fuse, noise_main, noise_concepts, masks, guidance, 0.0, 0.0, latents, next_main_in, next_concept_in,
               latents_f16)
    d.c_x, d.c_eps, d.a, d.b, d.c, d.d, d.input_scale = (float(v) for v in coeffs)
    if history is not None and (history.dtype != torch.float32 or not history.is_contiguous()
                                or history.numel() != 2 * d.fuse.HW * 4):
        raise ValueError("history must be a contiguous fp32 (2, h, w, 4) tensor")
    if noise is not None and (noise.dtype != torch.float16 or not noise.is_contiguous()
                              or noise.numel() != 2 * 4 * d.fuse.HW):
        raise ValueError("noise must be a contiguous fp16 (2, 4, h, w) tensor")
    d.history = _ptr(history)
    d.noise = _ptr(noise)
    d.store_x0 = int(bool(store_x0))
    L.check(L.load().omg_solver_step(C.byref(d), _stream()), "omg_solver_step")


def axpy(a, b, alpha=1.0, out=None):
    """out = a + alpha * b (fp16, same shape)."""
    _chk16(a)
    if out is None:
        out = torch.empty_like(a)
    L.check(L.load().omg_axpy(a.data_ptr(), b.data_ptr(), float(alpha), out.data_ptr(), a.numel(), _stream()),
            "omg_axpy")
    return out


def softmax_rows(x, scale=1.0):
    """In-place softmax(scale * x) over the last dimension of a 2-D fp16 or bf16 matrix (rows may be strided)."""
    dt = _op_dtype(x)
    assert x.dim() == 2 and x.stride(1) == 1
    name = "omg_softmax_rows_bf16" if dt == torch.bfloat16 else "omg_softmax_rows"
    L.check(getattr(L.load(), name)(_ptr(x), x.shape[0], x.shape[1], x.stride(0), float(scale), _stream()), name)
    return x


def ctx_mix(ctx, coef, out=None):
    _chk16(ctx)
    B, Lk, Cc = ctx.shape
    if out is None:
        out = torch.empty_like(ctx)
    L.check(L.load().omg_ctx_mix(ctx.data_ptr(), coef.data_ptr(), out.data_ptr(), B, Lk, Cc, _stream()),
            "omg_ctx_mix")
    return out


def _rows(t):
    """(B, H, W, C) view with unit channel stride and pixels in row-major order -> (B, H, W, row stride)."""
    B, H, W, Cc = t.shape
    assert t.stride(3) == 1 and t.stride(1) == t.stride(2) * W and t.stride(0) == t.stride(1) * H
    return B, H, W, t.stride(2)


def channel_op(x, scale=None, shift=None, act=L.CH_ACT_NONE, slope=None, addend=None, add_scale=1, act_after_add=False,
               out=None):
    """omg_channel_op over (B, H, W, C) fp16 views (rows may be strided along the channel axis): y = act(x * scale +
    shift) + addend, or act(x * scale + shift + addend) with act_after_add.  The addend is read at nearest
    (y // add_scale, x // add_scale).  x None reads as zero.  scale / shift / slope fp32 [C] or None."""
    ref = x if x is not None else addend
    _chk16(ref)
    if x is not None:
        B, H, W, ldx = _rows(x)
    else:
        B, Ha, Wa, _ = addend.shape
        H, W, ldx = Ha * add_scale, Wa * add_scale, 0
    Cc = ref.shape[3]
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=torch.float16, device=ref.device)
    _, _, _, ldy = _rows(out)
    ld_add = 0
    if addend is not None:
        _chk16(addend)
        assert addend.shape == (B, H // add_scale, W // add_scale, Cc)
        ld_add = _rows(addend)[3]
    for v in (scale, shift, slope):
        assert v is None or (v.is_cuda and v.dtype == torch.float32 and v.is_contiguous() and v.numel() >= Cc)
    L.check(L.load().omg_channel_op(_ptr(x), ldx, out.data_ptr(), ldy, _ptr(scale), _ptr(shift), _ptr(slope),
                                    _ptr(addend), ld_add, 0 if addend is None else add_scale, B, H, W, Cc, int(act),
                                    int(act_after_add), _stream()), "omg_channel_op")
    return out


def pool2d_out_size(n, k, stride, pad, ceil_mode):
    """Output extent of PyTorch / ONNX pooling along one axis."""
    o = (n + 2 * pad - k + (stride - 1 if ceil_mode else 0)) // stride + 1
    if ceil_mode and (o - 1) * stride >= n + pad:
        o -= 1
    return o


def pool2d(x, k, stride, pad=0, ceil_mode=False, count_include_pad=True, is_max=True, out=None):
    """omg_pool2d: max or average pooling of a contiguous (B, H, W, C) fp16 tensor, C % 8 == 0."""
    _chk16(x)
    assert x.is_contiguous()
    B, H, W, Cc = x.shape
    Ho, Wo = pool2d_out_size(H, k, stride, pad, ceil_mode), pool2d_out_size(W, k, stride, pad, ceil_mode)
    if out is None:
        out = torch.empty((B, Ho, Wo, Cc), dtype=torch.float16, device=x.device)
    assert out.shape == (B, Ho, Wo, Cc) and out.is_contiguous()
    L.check(L.load().omg_pool2d(x.data_ptr(), out.data_ptr(), B, H, W, Cc, k, stride, pad, int(ceil_mode),
                                int(count_include_pad), int(is_max), _stream()), "omg_pool2d")
    return out


def scrfd_detect(levels, num_anchors, det_thresh, det_scale, nms_thresh=0.4):
    """omg_scrfd_detect.  levels: list of (stride, fh, fw, scores, boxes, kps or None) with fp32 CUDA tensors of
    fh * fw * num_anchors rows (1 / 4 / 10 values each).  Returns the fp32 [n, 15] rows (box, score, 5 key-points) in
    NMS order (a device tensor: the count is read back once)."""
    d = L.ScrfdDesc()
    d.n_levels, d.num_anchors = len(levels), num_anchors
    T = 0
    for i, (s, fh, fw, sc, bx, kp) in enumerate(levels):
        for t in (sc, bx, kp):
            assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous())
        n = fh * fw * num_anchors
        assert sc.numel() == n and bx.numel() == 4 * n and (kp is None or kp.numel() == 10 * n)
        d.scores[i], d.boxes[i], d.kps[i] = sc.data_ptr(), bx.data_ptr(), _ptr(kp)
        d.stride[i], d.fh[i], d.fw[i] = s, fh, fw
        T += n
    dev = levels[0][3].device
    out = torch.empty((max(T, 1), 15), dtype=torch.float32, device=dev)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    d.det_thresh, d.nms_thresh, d.det_scale = float(det_thresh), float(nms_thresh), float(det_scale)
    d.out, d.max_out, d.count = out.data_ptr(), out.shape[0], count.data_ptr()
    L.check(L.load().omg_scrfd_detect(C.byref(d), _stream()), "omg_scrfd_detect")
    return out[: int(count.item())]


def text_gate(embed, guide, bias, nh, p, scale=None, out=None):
    """omg_text_gate (MaxSigmoidAttnBlock's gating): embed (B, H, W, Ce) and p (B, H, W, C2) fp16 views with row-major
    pixels (rows may be strided along the channel axis), guide fp32 (B, n, Ce), bias / scale fp32 [nh].  out (default:
    p, in place) receives p * gate."""
    _chk16(embed)
    _chk16(p)
    B, H, W, ld_e = _rows(embed)
    _, _, _, ld_p = _rows(p)
    out = p if out is None else out
    _chk16(out)
    _, _, _, ld_o = _rows(out)
    assert p.shape[:3] == embed.shape[:3] == out.shape[:3] and out.shape[3] == p.shape[3]
    Ce, C2 = embed.shape[3], p.shape[3]
    for v in (guide, bias, scale):
        assert v is None or (v.is_cuda and v.dtype == torch.float32 and v.is_contiguous())
    assert guide.shape[0] == B and guide.shape[2] == Ce
    L.check(L.load().omg_text_gate(embed.data_ptr(), ld_e, Ce, guide.data_ptr(), guide.shape[1], bias.data_ptr(),
                                   _ptr(scale), nh, p.data_ptr(), ld_p, out.data_ptr(), ld_o, C2, B, H * W, _stream()),
            "omg_text_gate")
    return out


def adaptive_maxpool(x, k, out, row0=0):
    """omg_adaptive_maxpool: AdaptiveMaxPool2d((k, k)) of x (B, H, W, C) (rows may be strided along the channel axis)
    into rows row0 .. row0 + k*k - 1 of out (B, rows, C) fp16 (unit channel stride)."""
    _chk16(x)
    _chk16(out)
    B, H, W, ldx = _rows(x)
    Cc = x.shape[3]
    assert out.dim() == 3 and out.shape[0] == B and out.shape[2] == Cc and out.stride(2) == 1
    L.check(L.load().omg_adaptive_maxpool(x.data_ptr(), ldx, B, H, W, Cc, k, out.data_ptr(), out.stride(0), out.stride(1),
                                          row0, _stream()), "omg_adaptive_maxpool")
    return out


def yolo_detect(levels, text, normalize_x, rows=None, nms=None):
    """omg_yolo_detect for one image.  levels: list of (stride, box (1, fh, fw, >=64) fp16, emb (1, fh, fw, >=E) fp16,
    cls_scale, cls_bias) with row-major pixels; text fp32 [nc, E] normalised.  Returns (rows [anchors, 6] fp32,
    detections [n, 6] fp32 or None).  nms: dict(conf, iou, max_wh, agnostic, max_det, gain, pad, clip) or None for
    pass (a) only."""
    assert text.is_cuda and text.dtype == torch.float32 and text.is_contiguous() and text.dim() == 2
    d = L.YoloDesc()
    d.n_levels, d.nc, d.E, d.normalize_x = len(levels), text.shape[0], text.shape[1], int(bool(normalize_x))
    T = 0
    for i, (s, box, emb, sc, bi) in enumerate(levels):
        _chk16(box)
        _chk16(emb)
        B, fh, fw, box_ld = _rows(box)
        assert B == 1 and emb.shape[:3] == box.shape[:3]
        d.box[i], d.emb[i], d.box_ld[i], d.emb_ld[i] = box.data_ptr(), emb.data_ptr(), box_ld, _rows(emb)[3]
        d.cls_scale[i], d.cls_bias[i] = float(sc), float(bi)
        d.stride[i], d.fh[i], d.fw[i] = s, fh, fw
        T += fh * fw
    dev = text.device
    if rows is None:
        rows = torch.empty((T, 6), dtype=torch.float32, device=dev)
    assert rows.shape == (T, 6) and rows.is_contiguous()
    d.text, d.rows = text.data_ptr(), rows.data_ptr()
    out = count = None
    if nms is not None:
        out = torch.empty((max(nms["max_det"], 1), 6), dtype=torch.float32, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        d.conf, d.iou, d.max_wh = float(nms["conf"]), float(nms["iou"]), float(nms.get("max_wh", 7680))
        d.agnostic, d.max_det = int(bool(nms.get("agnostic", False))), int(nms["max_det"])
        d.gain, (d.pad_x, d.pad_y), (d.clip_w, d.clip_h) = float(nms["gain"]), nms["pad"], nms["clip"]
        d.out, d.max_out, d.count = out.data_ptr(), out.shape[0], count.data_ptr()
    L.check(L.load().omg_yolo_detect(C.byref(d), _stream()), "omg_yolo_detect")
    return rows, None if out is None else out[: int(count.item())]


# ------------------------------------------------------------------ weight packing (host, once per model load)
def pack_conv3x3_weight(w):
    """torch Conv2d weight [N, C, 3, 3] -> [N, 9*C] with K order (ky, kx, c)."""
    N, Cc = w.shape[:2]
    return w.permute(0, 2, 3, 1).reshape(N, 9 * Cc).contiguous()


def pack_geglu_weight(w, b=None):
    """GEGLU proj Linear(c -> 8c): rows [value(4c) ; gate(4c)] -> interleaved (value_j, gate_j)."""
    n2 = w.shape[0] // 2
    wi = torch.stack([w[:n2], w[n2:]], dim=1).reshape(w.shape[0], w.shape[1]).contiguous()
    bi = None if b is None else torch.stack([b[:n2], b[n2:]], dim=1).reshape(-1).contiguous()
    return wi, bi
