"""CPU tests of the bf16 decode path: the bf16 GEMM descriptor is validated before any CUDA call (fake pointers, never
dereferenced), the new entry points are exported and bound, and the CLIs handle --decode."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from omg_b200 import _lib as L
    return L, L.load()


def _desc(L):
    """A descriptor that passes every check up to the first CUDA call: one 64-channel A view, N = 64."""
    d = L.GemmDesc()
    d.n_a, d.n_segs = 1, 1
    d.a[0] = L.View4(0x1000, 64, 16, 1, 1, 64, 64 * 16, 64 * 16)
    d.segs[0] = L.Seg(0, 0, 0, 0, 64, 0, 0)
    d.w, d.N, d.Ktot = 0x2000, 64, 64
    d.d = L.View4(0x3000, 64, 16, 1, 1, 64, 64 * 16, 64 * 16)
    d.dtype = L.DTYPE_BF16
    return d


def _err(lib, d):
    assert lib.omg_gemm(C.byref(d), None) == 1
    return lib.omg_last_error().decode()


def test_gemm_rejects_unknown_dtype():
    L, lib = _lib()
    d = _desc(L)
    d.dtype = 2
    assert "dtype=2 unsupported" in _err(lib, d)
    d.dtype = -1
    assert "dtype=-1 unsupported" in _err(lib, d)


@pytest.mark.parametrize("feature,message", [
    ("geglu", "bf16 supports only OMG_EPI_NONE (epilogue 1)"),
    ("silu", "bf16 supports only OMG_EPI_NONE (epilogue 2)"),
    ("quick_gelu", "bf16 supports only OMG_EPI_NONE (epilogue 3)"),
    ("gelu", "bf16 supports only OMG_EPI_NONE (epilogue 4)"),
    ("gelu_tanh", "bf16 supports only OMG_EPI_NONE (epilogue 5)"),
    ("relu", "bf16 supports only OMG_EPI_NONE (epilogue 6)"),
    ("rowvec", "bf16 does not support rowvec"),
    ("w2", "bf16 does not support a second weight matrix (w2)"),
    ("planes", "bf16 does not support weight planes"),
    ("ln_fold", "bf16 does not support the folded LayerNorm"),
    ("row_stats", "bf16 does not support row statistics"),
    ("col_stats", "bf16 does not support column statistics"),
    ("residual_f32", "bf16 does not support fp32 twins"),
    ("out_f32", "bf16 does not support fp32 twins"),
])
def test_bf16_gemm_rejects_unsupported_features(feature, message):
    L, lib = _lib()
    d = _desc(L)
    epi = {"geglu": L.EPI_GEGLU, "silu": L.EPI_SILU, "quick_gelu": L.EPI_QUICK_GELU, "gelu": L.EPI_GELU,
           "gelu_tanh": L.EPI_GELU_TANH, "relu": L.EPI_RELU}
    if feature in epi:
        d.epilogue = epi[feature]
    elif feature == "rowvec":
        d.rowvec, d.rowvec_ld = 0x4000, 64
    elif feature == "w2":
        d.w2, d.K2tot = 0x4000, 64
    elif feature == "planes":
        d.w_group_planes = d.n_col_groups = 2
        d.col_group_end[0] = 128
    elif feature == "ln_fold":
        d.row_stats_in, d.row_stats_parts, d.ln_dim, d.col_c1, d.col_c2 = 0x4000, 2, 64, 0x5000, 0x6000
    elif feature == "row_stats":
        d.row_stats_out = 0x4000
    elif feature == "col_stats":
        d.col_stats_out, d.col_stats_rb_total = 0x4000, 4
    elif feature == "residual_f32":
        d.residual_f32, d.residual_f32_ld = 0x4000, 64
    elif feature == "out_f32":
        d.out_f32, d.out_f32_ld = 0x4000, 64
    assert message in _err(lib, d)


def test_zeroed_descriptor_is_fp16():
    from omg_b200 import _lib as L
    assert L.GemmDesc().dtype == L.DTYPE_F16 == 0
    assert [f for f, _ in L.GemmDesc._fields_][-1] == "dtype"  # appended: earlier fields keep their offsets


def test_bf16_entry_points_are_exported_and_validate_first():
    L, lib = _lib()
    hdr = open(os.path.join(ROOT, "include", "omg_b200.h")).read()
    for name in ("omg_groupnorm_bf16", "omg_softmax_rows_bf16"):
        assert re.search(rf"\b{name}\s*\(", hdr) and name in L.SYMBOLS
        assert hasattr(C.CDLL(L.LIB_PATH), name)
    assert "OMG_DTYPE_BF16 = 1" in hdr and "OMG_DTYPE_F16 = 0" in hdr
    fake = C.c_void_p(0x1000)

    def err(rc):
        assert rc == 1
        return lib.omg_last_error().decode()

    assert "omg_softmax_rows_bf16: cols=12 must be a multiple of 8" in err(lib.omg_softmax_rows_bf16(fake, 4, 12, 16, 1.0, None))
    assert "omg_softmax_rows_bf16: scale must be positive" in err(lib.omg_softmax_rows_bf16(fake, 4, 16, 16, -1.0, None))
    assert "omg_groupnorm_bf16: bad channel split" in err(
        lib.omg_groupnorm_bf16(fake, 100, None, 0, 1, 16, fake, fake, 1e-6, 0, fake, fake, None))
    assert "omg_groupnorm_bf16: C=48 must be a multiple of 32" in err(
        lib.omg_groupnorm_bf16(fake, 48, None, 0, 1, 16, fake, fake, 1e-6, 0, fake, fake, None))


def test_ops_reject_cpu_and_mixed_operands():
    import torch
    from omg_b200 import ops
    with pytest.raises(ValueError):
        ops.linear(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        ops.softmax_rows(torch.zeros(2, 16, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        ops.groupnorm(torch.zeros(1, 4, 32, dtype=torch.bfloat16), torch.ones(32), torch.zeros(32), 1e-6, 0)


def _run_cli(script, *argv):
    return subprocess.run([sys.executable, os.path.join(ROOT, script), *argv], cwd=ROOT, capture_output=True, text=True,
                          timeout=300)


def test_lora_cli_decode_and_fp16_safe_vae_are_exclusive():
    r = _run_cli("inference_lora.py", "--decode", "--vae_fp16_safe", "/nonexistent")
    assert r.returncode != 0 and "--decode and --vae_fp16_safe are exclusive" in r.stderr


def _parse(script, argv):
    import importlib.util
    spec = importlib.util.spec_from_file_location("cli_" + script[:-3], os.path.join(ROOT, script))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    saved, sys.argv = sys.argv, [script, *argv]
    try:
        return mod, mod.parse_args()
    finally:
        sys.argv = saved


def test_cli_decode_flags_parse():
    mod, ns = _parse("inference_lora.py", ["--decode", "--vae_fp16_safe", "x"])
    with pytest.raises(SystemExit, match="exclusive"):
        mod.check_decode_flags(ns)
    mod.check_decode_flags(_parse("inference_lora.py", ["--decode"])[1])
    mod.check_decode_flags(_parse("inference_lora.py", ["--vae_fp16_safe", "x"])[1])
    _, ns = _parse("inference_instantid.py", ["--decode", "--synthetic", "--tiny"])
    assert ns.decode and ns.synthetic and ns.tiny
    assert not _parse("inference_instantid.py", [])[1].decode


def test_sam_flag_message_names_decode():
    from omg_b200.sam import check_sam_flags
    with pytest.raises(SystemExit, match="--decode"):
        check_sam_flags("1,2,3,4", "", decoded=False)
