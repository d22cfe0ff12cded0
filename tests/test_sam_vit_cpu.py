"""CPU checks of the original-SAM (ViT) attention: the fp32 oracle's decomposed relative-position bias against explicit
loops over its definition, window padding as bias tokens, the image-encoder topology read off a state dict, and the
omg_attention_relpos descriptor (C layout, rejections before any CUDA call)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _loop_bias(q, rel_h, rel_w, H, W):
    """B[q, k] = q . Rh[qh - kh + H - 1] + q . Rw[qw - kw + W - 1], by loops over the definition."""
    n = H * W
    out = torch.zeros(q.shape[0], n, n, dtype=torch.float64)
    for b in range(q.shape[0]):
        for i in range(n):
            qh, qw = divmod(i, W)
            for j in range(n):
                kh, kw = divmod(j, W)
                out[b, i, j] = q[b, i] @ rel_h[qh - kh + H - 1] + q[b, i] @ rel_w[qw - kw + W - 1]
    return out


@pytest.mark.parametrize("H,W", [(4, 5), (3, 3)])
def test_decomposed_rel_pos_equals_the_loop_definition(H, W):
    from oracle.sam_vit import add_decomposed_rel_pos
    g = torch.Generator().manual_seed(H * W)
    q = torch.randn(2, H * W, 8, generator=g, dtype=torch.float64)
    rh = torch.randn(2 * H - 1, 8, generator=g, dtype=torch.float64)
    rw = torch.randn(2 * W - 1, 8, generator=g, dtype=torch.float64)
    zero = torch.zeros(2, H * W, H * W, dtype=torch.float64)
    assert torch.allclose(add_decomposed_rel_pos(zero, q, rh, rw, (H, W), (H, W)), _loop_bias(q, rh, rw, H, W))


def test_decomposed_rel_pos_in_windows_uses_window_coordinates():
    """Windowed attention: the bias of a key depends on its position inside its window, not in the grid."""
    from oracle.sam_vit import add_decomposed_rel_pos, window_partition
    g = torch.Generator().manual_seed(1)
    ws, H, W, hd = 3, 5, 4, 4
    x = torch.randn(1, H, W, hd, generator=g, dtype=torch.float64)
    rh = torch.randn(2 * ws - 1, hd, generator=g, dtype=torch.float64)
    rw = torch.randn(2 * ws - 1, hd, generator=g, dtype=torch.float64)
    wins, (Hp, Wp) = window_partition(x, ws)
    assert (Hp, Wp) == (6, 6) and wins.shape == (4, ws, ws, hd)
    q = wins.reshape(4, ws * ws, hd)
    got = add_decomposed_rel_pos(torch.zeros(4, ws * ws, ws * ws, dtype=torch.float64), q, rh, rw, (ws, ws), (ws, ws))
    assert torch.allclose(got, _loop_bias(q, rh, rw, ws, ws))
    # padded positions of window_partition are zeros of the (normalised) input
    assert torch.equal(wins[3, 2], torch.zeros(ws, hd, dtype=torch.float64))


def test_padded_window_keys_are_bias_tokens_not_masked_keys():
    """A padded grid: the reference's padded keys are qkv(0) = the bias and take part in every softmax.  Masking them out
    instead gives a different output, so the kernel must not mask them."""
    from oracle.sam_vit import attention_block_attn
    g = torch.Generator().manual_seed(2)
    C, heads, ws, H, W = 16, 2, 4, 6, 7
    sd = {"attn.qkv.weight": torch.randn(3 * C, C, generator=g) * 0.3, "attn.qkv.bias": torch.randn(3 * C, generator=g),
          "attn.proj.weight": torch.randn(C, C, generator=g) * 0.3, "attn.proj.bias": torch.zeros(C),
          "attn.rel_pos_h": torch.randn(2 * ws - 1, C // heads, generator=g) * 0.2,
          "attn.rel_pos_w": torch.randn(2 * ws - 1, C // heads, generator=g) * 0.2}
    x = torch.randn(1, H, W, C, generator=g)
    ref = attention_block_attn(x, sd, "", heads, ws)
    pad = torch.zeros(1, 8, 8, dtype=torch.bool)
    pad[:, H:, :] = True
    pad[:, :, W:] = True
    keys_pad = pad.view(1, 2, 4, 2, 4).permute(0, 1, 3, 2, 4).reshape(4, 1, ws * ws)  # per window, per key
    keys_pad = keys_pad.repeat_interleave(heads, 0)

    def mask(a):
        return a.masked_fill(keys_pad, float("-inf"))

    masked = attention_block_attn(x, sd, "", heads, ws, mask_fn=mask)
    assert ref.shape == (1, H, W, C)
    assert (ref - masked).abs().max() > 1e-2


def _shape_sd(C, depth, hd, glob):
    """Image-encoder state dict with the checkpoint's key set and shapes (meta tensors: no memory)."""
    sd = {"patch_embed.proj.weight": torch.empty(C, 3, 16, 16, device="meta"), "pos_embed": torch.empty(1, 64, 64, C,
                                                                                                       device="meta")}
    for i in range(depth):
        n = 127 if i in glob else 27
        sd[f"blocks.{i}.attn.rel_pos_h"] = torch.empty(n, hd, device="meta")
        sd[f"blocks.{i}.attn.rel_pos_w"] = torch.empty(n, hd, device="meta")
        sd[f"blocks.{i}.attn.qkv.weight"] = torch.empty(3 * C, C, device="meta")
    return sd


@pytest.mark.parametrize("kind,C,depth,heads,glob", [("vit_b", 768, 12, 12, (2, 5, 8, 11)),
                                                      ("vit_l", 1024, 24, 16, (5, 11, 17, 23)),
                                                      ("vit_h", 1280, 32, 16, (7, 15, 23, 31))])
def test_topology_is_read_off_the_state_dict(kind, C, depth, heads, glob):
    from oracle.sam_vit import topology
    assert topology(_shape_sd(C, depth, C // heads, glob)) == (C, depth, heads, C // heads, glob)


# ------------------------------------------------------------------------------------------------------ C descriptor
FIELDS = ["qkv", "ld", "bs", "q_col0", "k_col0", "v_col0", "out", "out_ld", "out_bs", "out_col0", "B", "H", "W", "heads",
          "head_dim", "window", "rel_pos_h", "rel_h_len", "rel_pos_w", "rel_w_len", "k_bias", "v_bias", "scale"]


def test_relpos_descriptor_ctypes_layout_matches_c():
    from omg_b200 import _lib as L
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    assert [f[0] for f in L.AttnRelposDesc._fields_] == FIELDS
    src = "#include <stddef.h>\n#include <stdio.h>\n#include \"omg_b200.h\"\nint main(void) {\n"
    src += '    printf("%zu\\n", sizeof(omg_attn_relpos_desc));\n'
    src += "".join(f'    printf("%zu\\n", offsetof(omg_attn_relpos_desc, {f}));\n' for f in FIELDS)
    src += "    return 0;\n}\n"
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "layout.c"), "w") as f:
            f.write(src)
        exe = os.path.join(tmp, "layout")
        subprocess.run([cc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                        os.path.join(tmp, "layout.c"), "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(L.AttnRelposDesc)] + [getattr(L.AttnRelposDesc, f).offset for f in FIELDS]
    assert got == want


def _valid_desc(L, hd=80, window=14, H=64, W=64):
    d = L.AttnRelposDesc()
    heads = 2
    d.qkv, d.ld, d.bs, d.q_col0, d.k_col0, d.v_col0 = 0x1000, 3 * heads * hd, H * W * 3 * heads * hd, 0, heads * hd, \
        2 * heads * hd
    d.out, d.out_ld, d.out_bs, d.out_col0 = 0x2000, heads * hd, H * W * heads * hd, 0
    d.B, d.H, d.W, d.heads, d.head_dim, d.window = 1, H, W, heads, hd, window
    S = (window, window) if window else (H, W)
    d.rel_pos_h, d.rel_h_len, d.rel_pos_w, d.rel_w_len = 0x3000, 2 * S[0] - 1, 0x4000, 2 * S[1] - 1
    d.k_bias, d.v_bias, d.scale = 0x5000, 0x6000, hd ** -0.5
    return d


def test_relpos_rejections_happen_before_any_cuda_call():
    """Each bad descriptor is refused by validation (its own message) - none of these calls reaches a CUDA API, so they
    run on a machine without a GPU; pointers are never dereferenced."""
    from omg_b200 import _lib as L
    lib = L.load()

    def err(d):
        assert lib.omg_attention_relpos(None if d is None else C.byref(d), None) == 1
        return lib.omg_last_error().decode()

    assert "null descriptor" in err(None)
    cases = [
        (dict(head_dim=96), "head_dim 96 unsupported"),
        (dict(heads=0), "empty problem"),
        (dict(window=65), "window 65 out of range"),
        (dict(window=-1), "window -1 out of range"),
        (dict(rel_h_len=29), "rel_pos_h has 29 rows, expected 2 * 14 - 1 = 27"),
        (dict(rel_w_len=127), "rel_pos_w has 127 rows, expected 2 * 14 - 1 = 27"),
        (dict(qkv=None), "null pointer"),
        (dict(rel_pos_w=None), "null pointer"),
        (dict(k_bias=None), "k_bias and v_bias"),
        (dict(v_bias=None), "k_bias and v_bias"),
        (dict(qkv=0x1008), "qkv rows must be 16 B aligned"),
        (dict(ld=3 * 2 * 80 + 4), "qkv rows must be 16 B aligned"),
        (dict(rel_pos_h=0x3004), "rel-pos tables must be 16 B aligned"),
        (dict(out_col0=4), "output must be 16 B aligned"),
        (dict(v_col0=2 * 160 + 8), "v head window [328, 488) does not fit its row of 480"),
        (dict(out_ld=152), "out head window [0, 160) does not fit its row of 152"),
        (dict(q_col0=-8), "q head window [-8, 152)"),
    ]
    for change, msg in cases:
        d = _valid_desc(L)
        for k, v in change.items():
            setattr(d, k, v)
        assert msg in err(d), (change, lib.omg_last_error())
    # global attention: grid at most 64 x 64, tables 2H - 1 / 2W - 1
    d = _valid_desc(L, window=0, H=65, W=64)
    assert "global attention over a 65 x 64 grid" in err(d)
    d = _valid_desc(L, window=0, H=32, W=48)
    d.rel_h_len = 127
    assert "rel_pos_h has 127 rows, expected 2 * 32 - 1 = 63" in err(d)
    d = _valid_desc(L, window=0, H=32, W=48)
    d.rel_w_len = 63
    assert "rel_pos_w has 63 rows, expected 2 * 48 - 1 = 95" in err(d)
    # the biases are optional when no window is padded (70 = 5 windows of 14) and in global attention
    for d in (_valid_desc(L, H=70, W=70), _valid_desc(L, window=0)):
        d.k_bias = d.v_bias = None
        d.out_col0 = 4       # stop at a later check: the bias check passed
        assert "output must be 16 B aligned" in err(d)


def test_ops_wrapper_has_no_cpu_path():
    from omg_b200 import ops
    z = torch.zeros(1, 16, 3 * 64, dtype=torch.float16)
    t = torch.zeros(7, 64, dtype=torch.float16)
    with pytest.raises(ValueError):
        ops.attention_relpos(z, 4, 4, 1, 64, t, t)
