"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads, and exports every
symbol include/lvb200.h declares (no compute calls - there is no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "lvb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(lv_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_hot_path():
    syms = declared_symbols()
    for must in ["lv_attn_fwd", "lv_rmsnorm", "lv_rope", "lv_swiglu", "lv_gemm_bias_act", "lv_patch_embed",
                 "lv_embed_scatter", "lv_pixel_shuffle", "lv_row_gather", "lv_last_error"]:
        assert must in syms


def test_library_exports_every_declared_symbol(lib_built):
    lib = ctypes.CDLL(lib_built)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"liblvb200.so does not export: {missing}"


def test_python_binding_covers_every_declared_symbol(lib_built):
    from long_vita_b200 import _lib

    assert sorted(_lib.SIGNATURES) == declared_symbols()
    handle = _lib.lib()
    assert handle.lv_version() >= 1000
    assert handle.lv_last_error() == b""


def test_attn_params_struct_matches_header():
    from long_vita_b200._lib import AttnParams

    # 5 pointers + 6 int64 + 4*3 int64 + float + int32 + int64 + 2 int64 + int64
    assert ctypes.sizeof(AttnParams) == 5 * 8 + 6 * 8 + 12 * 8 + 4 + 4 + 8 + 16 + 8


def test_bad_arguments_fail_loudly_without_a_gpu(lib_built):
    from long_vita_b200 import _lib

    h = _lib.lib()
    rc = h.lv_swiglu(None, None, 4, 16, None)
    assert rc == -1 and b"null pointer" in h.lv_last_error()
    rc = h.lv_gemm_bias_act(1, 1, None, 1, 4, 8, 7, 7, 7, 8, 0, None)
    assert rc == -1 and b"multiples of 8" in h.lv_last_error()


def test_ops_refuse_cpu_tensors(lib_built):
    import torch

    from long_vita_b200 import ops

    x = torch.zeros(4, 16, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.swiglu(x)


def _attn_params(**kw):
    from long_vita_b200._lib import AttnParams

    p = AttnParams()
    p.q = p.k = p.v = p.out = 0x1000                    # never dereferenced: every case below fails validation first
    p.lse = None
    p.batch, p.sq, p.sk, p.hq, p.hkv, p.d = 1, 256, 256, 8, 2, 128
    for arr, row in ((p.q_strides, 8 * 128), (p.k_strides, 2 * 128), (p.v_strides, 2 * 128), (p.o_strides, 8 * 128)):
        arr[0], arr[1], arr[2] = 256 * row, row, 128
    p.scale, p.causal, p.q_seg_len, p.kv_pos0 = 0.088, 1, 256, 0
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("kw,msg", [
    (dict(d=96), b"head_dim 96 not supported"),
    (dict(hq=7), b"not a multiple of hkv"),
    (dict(sq=0), b"empty shape"),
    (dict(q=None), b"null tensor pointer"),
    (dict(q_seg_len=300), b"out of range"),
    (dict(q_seg_len=100), b"q_seg_len % 128 == 0"),
    (dict(scale=0.0), b"must be finite and > 0"),
    (dict(scale=-0.1), b"must be finite and > 0"),
    (dict(scale=float("nan")), b"must be finite and > 0"),
    (dict(scale=float("inf")), b"must be finite and > 0"),
])
def test_attention_argument_errors_have_the_documented_code_and_text(lib_built, kw, msg):
    """INTEGRATION.md section 4: every entry point returns a negative LV_E* code and sets lv_last_error()."""
    from long_vita_b200 import _lib

    h = _lib.lib()
    p = _attn_params(**kw)
    rc = h.lv_attn_fwd(ctypes.byref(p), None)
    assert rc == -1 and msg in h.lv_last_error(), h.lv_last_error()
    with pytest.raises(RuntimeError, match="lv_attn_fwd failed"):
        _lib.check(rc, "lv_attn_fwd")
    if "scale" in kw:
        # the document-masked and context-parallel forwards and the backward refuse the same scales
        from long_vita_b200._lib import AttnBwdParams, AttnDocs, CpParams

        assert h.lv_attn_docs_fwd(ctypes.byref(p), ctypes.byref(AttnDocs()), None) == -1 and msg in h.lv_last_error()
        assert h.lv_attn_cp_fwd(ctypes.byref(p), ctypes.byref(CpParams()), None) == -1 and msg in h.lv_last_error()
        b = AttnBwdParams()
        b.fwd = p
        b.fwd.lse = 0x1000
        b.d_out = b.dq = b.dk = b.dv = b.delta_ws = 0x1000
        assert h.lv_attn_bwd(ctypes.byref(b), None) == -1 and msg in h.lv_last_error()
        assert h.lv_attn_docs_bwd(ctypes.byref(b), ctypes.byref(AttnDocs()), None) == -1 and msg in h.lv_last_error()


def test_backward_and_gemm_argument_errors(lib_built):
    from long_vita_b200 import _lib
    from long_vita_b200._lib import AttnBwdParams

    h = _lib.lib()
    assert h.lv_attn_bwd_ws_bytes(1, 40, 16384) == 40 * 16384 * 4
    b = AttnBwdParams()
    assert h.lv_attn_bwd(ctypes.byref(b), None) == -1 and b"required" in h.lv_last_error()
    # the backward takes the forward's size limits; each case fails validation before any pointer is used
    for kw, msg in ((dict(sq=1 << 30, q_seg_len=1 << 30), b"sequence too long"),
                    (dict(sk=1 << 30), b"sequence too long"),
                    (dict(sq=(1 << 30) - 1, q_seg_len=(1 << 30) - 1, batch=256), b"too many work items"),     # dQ pass
                    (dict(sq=128, q_seg_len=128, sk=1 << 29, hq=8, hkv=8, batch=64), b"too many work items"),  # dK/dV pass
                    (dict(q_seg_len=100), b"bad query segmentation"),
                    (dict(d=96), b"head_dim 96 not supported")):
        b = AttnBwdParams()
        b.fwd = _attn_params(**kw)
        b.fwd.lse = 0x1000
        b.d_out = b.dq = b.dk = b.dv = b.delta_ws = 0x1000
        assert h.lv_attn_bwd(ctypes.byref(b), None) == -1 and msg in h.lv_last_error(), (kw, h.lv_last_error())
    b = AttnBwdParams()
    b.fwd = _attn_params()
    b.fwd.lse = 0x1000
    b.d_out = b.dq = b.dk = b.dv = b.delta_ws = 0x1000
    b.fwd.sq, b.fwd.q_seg_len, b.fwd.batch = 256, 256, 1 << 23   # 2^23 * 8 heads * 2 tiles = 2^27 items: within limits
    b.dq_strides[0] = 12                                         # ... so the stride check is what refuses it
    assert h.lv_attn_bwd(ctypes.byref(b), None) == -1 and b"multiples of 8" in h.lv_last_error()
    assert h.lv_gemm_bias_act(1, 1, None, 1, 4, 24, 8, 8, 8, 24, 3, None) == -1 and b"SwiGLU" in h.lv_last_error()
    assert h.lv_gemm_bias_act(1, 1, None, 1, 4, 16, 8, 8, 8, 16, 7, None) == -1 and b"unknown activation" in h.lv_last_error()


def test_image_tiling_argument_errors(lib_built):
    import torch

    from long_vita_b200 import _lib
    from long_vita_b200 import preprocess as PP

    h = _lib.lib()
    assert h.lv_image_tiles_ws_bytes(300, 896) == 300 * 896 * 3
    args = lambda oh, ow, base=0: (1, 1, 1, 1, 1, 1, 5, 1, 1, 1, 5, 300, 200, oh, ow, 448, base, 1, 1, None)   # noqa: E731
    assert h.lv_image_tiles_preprocess(*args(448, 900)) == -1 and b"not a grid of 448-pixel tiles" in h.lv_last_error()
    assert h.lv_image_tiles_preprocess(*args(0, 448)) == -1 and b"empty shape" in h.lv_last_error()
    assert h.lv_image_tiles_preprocess(*args(448, 448, -1)) == -1 and b"empty shape" in h.lv_last_error()
    assert h.lv_image_tiles_preprocess(None, 1, 1, 1, 1, 1, 5, 1, 1, 1, 5, 300, 200, 448, 448, 448, 0, 1, 1, None) == -1
    assert b"null pointer" in h.lv_last_error()
    with pytest.raises(ValueError, match="CUDA uint8"):
        PP.preprocess_image_dynamic(torch.zeros(8, 8, 3, dtype=torch.uint8))


def test_missing_extension_fails_loudly(monkeypatch):
    """No CPU / PyTorch fallback: without liblvb200.so every operator raises, naming the build command."""
    from long_vita_b200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/liblvb200.so")
    with pytest.raises(RuntimeError, match="is missing"):
        _lib.lib()
    from long_vita_b200 import ops

    with pytest.raises(RuntimeError):
        ops.launch_count()
    monkeypatch.undo()
    assert _lib.lib().lv_version() >= 1000


def test_product_package_never_imports_the_oracle():
    """oracle/ is test infrastructure: only tests/, __graft_entry__.smoke() and bench.py's CPU legs may use it."""
    import ast

    pkg = os.path.join(ROOT, "long-vita_b200")
    offenders = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if not f.endswith(".py"):
                continue
            tree = ast.parse(open(os.path.join(dirpath, f)).read())
            for node in ast.walk(tree):
                names = []
                if isinstance(node, ast.Import):
                    names = [a.name for a in node.names]
                elif isinstance(node, ast.ImportFrom) and node.level == 0:
                    names = [node.module or ""]
                if any(n == "oracle" or n.startswith("oracle.") or n == "tests" or n.startswith("tests.") for n in names):
                    offenders.append(os.path.join(dirpath, f))
    assert not offenders, offenders


def test_context_parallel_argument_errors(lib_built):
    from long_vita_b200 import _lib
    from long_vita_b200._lib import CpParams

    h = _lib.lib()
    a = _attn_params()
    c = CpParams()
    c.rank, c.cp, c.seq_total = 0, 9, 4096
    assert h.lv_attn_cp_fwd(ctypes.byref(a), ctypes.byref(c), None) == -1 and b"bad rank" in h.lv_last_error()
    c.cp = 2
    c.seq_total = 4098
    assert h.lv_attn_cp_fwd(ctypes.byref(a), ctypes.byref(c), None) == -1 and b"not divisible by 2*cp" in h.lv_last_error()
    c.seq_total = 4 * 100
    assert h.lv_attn_cp_fwd(ctypes.byref(a), ctypes.byref(c), None) == -1 and b"multiple of 128" in h.lv_last_error()
    c.seq_total = 4 * 128
    assert h.lv_attn_cp_fwd(ctypes.byref(a), ctypes.byref(c), None) == -1 and b"staging buffers" in h.lv_last_error()
