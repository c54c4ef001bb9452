"""The C calls the operator wrappers of `ops` make, and the arguments they refuse, on CPU.

The C entry points cannot see tensor extents, so each wrapper hands its tensors over in the form the kernel reads and
checks what the kernel will read.  A stub library records every `lv_*` call, so no kernel runs: the table below pins the
call (symbol, pointers, sizes, strides, flags) each wrapper makes on contiguous inputs and on the strided views it
reads in place, every mismatch the wrappers check raises ValueError before anything is recorded, and the GEMM operand
rule maps each layout to the reading or the copy the kernel needs.
"""
import types
from unittest.mock import ANY

import pytest
import torch

from long_vita_b200 import ops


class _Lib:
    """Records each `lv_*` launch as (symbol, arguments without the stream) and reports success."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name.endswith(("_partials", "_ws_bytes")):        # size queries, no stream and nothing launched
            return lambda *a: 2
        return lambda *a: self.calls.append((name,) + a[:-1]) or 0


@pytest.fixture
def lib(monkeypatch):
    fake = _Lib()
    monkeypatch.setattr(ops._lib, "lib", lambda: fake)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_need_cuda_bf16", lambda *ts: None)
    monkeypatch.setattr(ops, "_need_cuda", lambda t, dtype: None)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
    return fake


def _bf16(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def _f32(*shape):
    return torch.zeros(*shape, dtype=torch.float32)


def _i64(*shape):
    return torch.zeros(*shape, dtype=torch.int64)


def P(t):
    return t.data_ptr()


# ------------------------------------------------------------------------------------------------
# recorded calls: each case calls one wrapper and returns the call it must record
# ------------------------------------------------------------------------------------------------
def _rmsnorm():
    x, w, r = _bf16(3, 5, 64), _bf16(64), _bf16(15, 64)
    y, s = ops.rmsnorm(x, w, 1e-5, residual=r)
    return ("lv_rmsnorm", P(x), P(r), P(w), P(y), P(s), 15, 64, 1e-5)


def _layernorm():
    x, w, b = _bf16(4, 32), _bf16(32), _bf16(32)
    y = ops.layernorm(x, w, b, 1e-6)
    return ("lv_layernorm", P(x), P(w), P(b), P(y), 4, 32, 1e-6)


def _rope_table():
    pos, inv = _i64(7), _f32(32)
    cos, sin = ops.rope_table(pos, inv)
    return ("lv_rope_table", P(pos), P(inv), P(cos), P(sin), 7, 64)


def _rope_strided_in_place():
    qkv = _bf16(6, 3 * 4 * 64)
    q = qkv[:, : 4 * 64].view(6, 4, 64)                  # a column slice of the fused QKV output, rotated in place
    cos, sin = _bf16(6, 64), _bf16(6, 64)
    ops.rope(q, cos, sin, out=q)
    return ("lv_rope", P(qkv), P(qkv), P(cos), P(sin), 6, 4, 64, 3 * 4 * 64, 64, 3 * 4 * 64, 64)


def _swiglu():
    gu = _bf16(2, 3, 32)
    h = ops.swiglu(gu)
    return ("lv_swiglu", P(gu), P(h), 6, 16)


def _bias_gelu():
    x, b = _bf16(5, 48), _bf16(48)
    y = ops.bias_gelu(x, b, "tanh")
    return ("lv_bias_gelu", P(x), P(b), P(y), 5, 48, 1)


def _ls_residual():
    x, y, ls, b = _bf16(2, 4, 16), _bf16(8, 16), _bf16(16), _bf16(16)
    o = ops.ls_residual(x, y, ls, b)
    return ("lv_ls_residual", P(x), P(y), P(b), P(ls), P(o), 8, 16)


def _pixel_shuffle():
    x = _bf16(2, 1 + 16, 8)
    o = ops.pixel_shuffle(x, 4, True)
    return ("lv_pixel_shuffle", P(x), P(o), 2, 4, 8, 1)


def _embed_scatter():
    ids, table, feat, dst, src = _i64(1, 9), _bf16(20, 16), _bf16(3, 16), _i64(2), _i64(2)
    o = ops.embed_scatter(ids, table, feat, dst, src)
    return ("lv_embed_scatter", P(ids), P(table), 20, P(feat), P(src), P(dst), 2, P(o), 9, 16)


def _row_gather():
    x, idx = _bf16(10, 16), _i64(4)
    o = ops.row_gather(x, idx)
    return ("lv_row_gather", P(x), P(idx), P(o), 4, 16)


def _row_scatter_zero():
    x, idx = _bf16(4, 16), _i64(4)
    o = ops.row_scatter_zero(x, idx, 10)
    return ("lv_row_scatter_zero", P(x), P(idx), P(o), 4, 10, 16)


def _ce_accumulate_strided_logits():
    buf, labels = _bf16(6, 40), _i64(6)
    run_max, run_sum, tgt = _f32(6), _f32(6), _f32(6)
    ops.ce_accumulate(buf[:, :32], labels, run_max, run_sum, tgt, 64)
    return ("lv_ce_accumulate", P(buf), 40, P(labels), P(run_max), P(run_sum), P(tgt), 6, 32, 64)


def _ce_grad_strided_logits():
    buf, labels, lse, dloss = _bf16(6, 40), _i64(6), _f32(6), _f32(6)
    ops.ce_grad(buf[:, :32], labels, lse, dloss, 0)
    return ("lv_ce_grad", P(buf), 40, P(buf), 40, P(labels), P(lse), P(dloss), 6, 32, 0)


def _decode_merge():
    o, lse = _bf16(3, 2, 4, 64), _f32(3, 4, 2)
    out = ops.decode_merge(o, lse)
    return ("lv_attn_decode_merge", P(o), P(lse), P(out), None, 3, 2, 4, 64)


def _rmsnorm_bwd():
    x, w, dy, a = _bf16(6, 32), _bf16(32), _bf16(2, 3, 32), _bf16(6, 32)
    dx, _ = ops.rmsnorm_bwd(x, w, dy, 1e-6, add_in=a)
    return ("lv_rmsnorm_bwd", P(x), P(w), P(dy), P(a), P(dx), ANY, 6, 32, 1e-6)


def _swiglu_bwd():
    gu, dh = _bf16(5, 32), _bf16(5, 16)
    d = ops.swiglu_bwd(gu, dh)
    return ("lv_swiglu_bwd", P(gu), P(dh), P(d), 5, 16)


def _layernorm_bwd():
    x, w, dy = _bf16(4, 32), _bf16(32), _bf16(4, 32)
    ops.layernorm_bwd(x, w, dy, 1e-6, need_dx=False)
    return ("lv_layernorm_bwd", P(x), P(w), P(dy), None, None, ANY, ANY, 4, 32, 1e-6)


def _gelu_bwd():
    pre, dy = _bf16(3, 24), _bf16(3, 24)
    dx = ops.gelu_bwd(pre, dy)
    return ("lv_gelu_bwd", P(pre), P(dy), P(dx), 3, 24, 0)


def _ls_residual_bwd():
    dout, y, ls = _bf16(3, 16), _bf16(3, 16), _bf16(16)
    dy, _ = ops.ls_residual_bwd(dout, y, ls)
    return ("lv_ls_residual_bwd", P(dout), P(y), P(ls), P(dy), ANY, 3, 16)


def _pixel_shuffle_bwd():
    d = _bf16(2, 4, 32)
    dx = ops.pixel_shuffle_bwd(d, 4, True)
    return ("lv_pixel_shuffle_bwd", P(d), P(dx), 2, 4, 8, 1)


def _patch_im2col():
    img = _bf16(2, 3, 28, 28)
    col = ops.patch_im2col(img, 14, 640)
    return ("lv_patch_im2col", P(img), P(col), 2, 28, 14, 640)


def _patch_embed():
    img, w, b, cls, pos = _bf16(2, 3, 28, 28), _bf16(16, 640), _bf16(16), _bf16(1, 1, 16), _bf16(5, 16)
    out = ops.patch_embed(img, w, b, cls, pos, 14)
    return ("lv_patch_embed", P(img), P(w), P(b), P(cls), P(pos), P(out), ANY, 2, 28, 14, 16)


def _linear_wgrad_accumulate_row_slices():
    dy, xs, mg = _bf16(13, 48), _bf16(13, 72), _f32(96, 64)
    ops.linear_wgrad_accumulate(dy, xs[:, :64], mg[48:])
    return ("lv_gemm_wgrad_acc_f32", P(dy), P(xs), P(mg) + 48 * 64 * 4, 48, 64, 13, 48, 72, 64, 1, 1)


CALLS = [_rmsnorm, _layernorm, _rope_table, _rope_strided_in_place, _swiglu, _bias_gelu, _ls_residual, _pixel_shuffle,
         _embed_scatter, _row_gather, _row_scatter_zero, _ce_accumulate_strided_logits, _ce_grad_strided_logits,
         _decode_merge, _rmsnorm_bwd, _swiglu_bwd, _layernorm_bwd, _gelu_bwd, _ls_residual_bwd, _pixel_shuffle_bwd,
         _patch_im2col, _patch_embed, _linear_wgrad_accumulate_row_slices]


@pytest.mark.parametrize("case", CALLS, ids=[c.__name__.strip("_") for c in CALLS])
def test_wrapper_records_the_expected_call(lib, case):
    want = case()
    assert lib.calls == [want]


# ------------------------------------------------------------------------------------------------
# refused arguments: ValueError naming the wrapper and the argument, nothing launched
# ------------------------------------------------------------------------------------------------
x64, w64 = _bf16(4, 64), _bf16(64)
REFUSED = [
    ("rmsnorm weight", lambda: ops.rmsnorm(x64, _bf16(32)), "rmsnorm: weight"),
    ("rmsnorm residual", lambda: ops.rmsnorm(x64, w64, residual=_bf16(3, 64)), "rmsnorm: residual"),
    ("layernorm weight", lambda: ops.layernorm(x64, _bf16(63), None), "layernorm: weight"),
    ("layernorm bias", lambda: ops.layernorm(x64, w64, _bf16(65)), "layernorm: bias"),
    ("bias_gelu bias", lambda: ops.bias_gelu(x64, _bf16(8)), "bias_gelu: bias"),
    ("ls_residual y", lambda: ops.ls_residual(x64, _bf16(5, 64)), "ls_residual: y"),
    ("ls_residual ls", lambda: ops.ls_residual(x64, x64, _bf16(32)), "ls_residual: ls"),
    ("ls_residual bias", lambda: ops.ls_residual(x64, x64, None, _bf16(2, 64)), "ls_residual: bias"),
    ("linear bias", lambda: ops.linear(x64, _bf16(16, 64), _bf16(8)), "linear: bias"),
    ("linear weight", lambda: ops.linear(x64, _bf16(16, 72)), "linear: weight"),
    ("patch_embed bias", lambda: ops.patch_embed(_bf16(1, 3, 28, 28), _bf16(16, 640), _bf16(8), None, _bf16(4, 16), 14),
     "patch_embed: bias"),
    ("patch_embed cls", lambda: ops.patch_embed(_bf16(1, 3, 28, 28), _bf16(16, 640), None, _bf16(8), _bf16(5, 16), 14),
     "patch_embed: cls"),
    ("patch_embed pos", lambda: ops.patch_embed(_bf16(1, 3, 28, 28), _bf16(16, 640), None, _bf16(16), _bf16(4, 16), 14),
     "patch_embed: pos"),
    ("patch_embed w_pad", lambda: ops.patch_embed(_bf16(1, 3, 28, 28), _bf16(16, 588), None, None, _bf16(4, 16), 14),
     "patch_embed: w_pad"),
    ("rmsnorm_bwd dy", lambda: ops.rmsnorm_bwd(x64, w64, _bf16(2, 64)), "rmsnorm_bwd: dy"),
    ("rmsnorm_bwd add_in", lambda: ops.rmsnorm_bwd(x64, w64, x64, add_in=_bf16(8, 64)), "rmsnorm_bwd: add_in"),
    ("rmsnorm_bwd weight", lambda: ops.rmsnorm_bwd(x64, _bf16(60), x64), "rmsnorm_bwd: weight"),
    ("swiglu_bwd dh", lambda: ops.swiglu_bwd(x64, _bf16(4, 64)), "swiglu_bwd: dh"),
    ("layernorm_bwd dy", lambda: ops.layernorm_bwd(x64, w64, _bf16(3, 64)), "layernorm_bwd: dy"),
    ("layernorm_bwd add_in", lambda: ops.layernorm_bwd(x64, w64, x64, add_in=_bf16(64)), "layernorm_bwd: add_in"),
    ("gelu_bwd dy", lambda: ops.gelu_bwd(x64, _bf16(4, 32)), "gelu_bwd: dy"),
    ("ls_residual_bwd dout", lambda: ops.ls_residual_bwd(_bf16(5, 64), x64, w64), "ls_residual_bwd: dout"),
    ("ls_residual_bwd ls", lambda: ops.ls_residual_bwd(x64, x64, _bf16(16)), "ls_residual_bwd: ls"),
    ("pixel_shuffle hw", lambda: ops.pixel_shuffle(_bf16(2, 17, 8), 4, False), "pixel_shuffle: x"),
    ("pixel_shuffle_bwd hw", lambda: ops.pixel_shuffle_bwd(_bf16(2, 9, 32), 4, True), "pixel_shuffle_bwd: dout"),
    ("ce_accumulate int32 labels", lambda: ops.ce_accumulate(_bf16(6, 32), torch.zeros(6, dtype=torch.int32), _f32(6),
                                                             _f32(6), _f32(6), 0), "ce_accumulate: labels"),
    ("ce_accumulate short labels", lambda: ops.ce_accumulate(_bf16(6, 32), _i64(5), _f32(6), _f32(6), _f32(6), 0),
     "ce_accumulate: labels"),
    ("ce_accumulate bf16 run_sum", lambda: ops.ce_accumulate(_bf16(6, 32), _i64(6), _f32(6), _bf16(6), _f32(6), 0),
     "ce_accumulate: run_sum"),
    ("ce_accumulate strided tgt", lambda: ops.ce_accumulate(_bf16(6, 32), _i64(6), _f32(6), _f32(6), _f32(12)[::2], 0),
     "ce_accumulate: tgt"),
    ("ce_grad int32 labels", lambda: ops.ce_grad(_bf16(6, 32), torch.zeros(6, dtype=torch.int32), _f32(6), _f32(6), 0),
     "ce_grad: labels"),
    ("ce_grad lse", lambda: ops.ce_grad(_bf16(6, 32), _i64(6), _f32(5), _f32(6), 0), "ce_grad: lse"),
    ("ce_grad bf16 dloss", lambda: ops.ce_grad(_bf16(6, 32), _i64(6), _f32(6), _bf16(6), 0), "ce_grad: dloss"),
    ("embed_scatter src_idx", lambda: ops.embed_scatter(_i64(9), _bf16(20, 16), _bf16(3, 16), _i64(2), _i64(3)),
     "embed_scatter: src_idx"),
    ("decode_merge lse_part", lambda: ops.decode_merge(_bf16(3, 2, 4, 64), _f32(3, 2, 4, 2)), "decode_merge: lse_part"),
    ("attention_bwd lse", lambda: ops.attention_bwd(_bf16(1, 128, 4, 64), _bf16(1, 128, 4, 64), _bf16(1, 128, 2, 64),
                                                    _bf16(1, 128, 2, 64), _bf16(1, 128, 4, 64), _f32(1, 128, 4),
                                                    causal=True), "attention_bwd: lse"),
    ("rope 2-D x", lambda: ops.rope(_bf16(6, 64), _bf16(6, 64), _bf16(6, 64)), "rope: x"),
    ("rope strided last dim", lambda: ops.rope(_bf16(6, 4, 128)[..., ::2], _bf16(6, 64), _bf16(6, 64)), "rope: x"),
    ("rope out", lambda: ops.rope(_bf16(6, 4, 64), _bf16(6, 64), _bf16(6, 64), out=_bf16(6, 2, 64)), "rope: out"),
    ("rope cos rows", lambda: ops.rope(_bf16(6, 4, 64), _bf16(1, 64), _bf16(6, 64)), "rope: cos"),
    ("rope sin dim", lambda: ops.rope(_bf16(6, 4, 64), _bf16(6, 64), _bf16(6, 32)), "rope: sin"),
    ("linear_wgrad_accumulate tokens", lambda: ops.linear_wgrad_accumulate(_bf16(8, 16), _bf16(9, 32), _f32(16, 32)),
     "linear_wgrad_accumulate: dY has 8"),
]


@pytest.mark.parametrize("call,match", [r[1:] for r in REFUSED], ids=[r[0] for r in REFUSED])
def test_mismatched_argument_raises_before_any_launch(lib, call, match):
    with pytest.raises(ValueError, match=match):
        call()
    assert lib.calls == []


# ------------------------------------------------------------------------------------------------
# the GEMM operand rule
# ------------------------------------------------------------------------------------------------
def _unaligned():
    buf = _bf16(24 * 64 + 4)
    return buf[4 : 4 + 24 * 64].view(24, 64)           # 8 bytes into its buffer


OPERANDS = [
    # name, operand [rows, K], mn_ok, expected (read in place, mn_major, leading dimension)
    ("contiguous", lambda: _bf16(24, 64), True, (True, False, 64)),
    ("row-strided", lambda: _bf16(24, 80)[:, :64], True, (True, False, 80)),
    ("transposed, column stride 24", lambda: _bf16(64, 24).t(), True, (True, True, 24)),
    ("transposed, refused as MN-major", lambda: _bf16(64, 24).t(), False, (False, False, 64)),
    ("transposed, column stride 20", lambda: _bf16(64, 20).t(), True, (False, False, 64)),
    ("unaligned start", _unaligned, True, (False, False, 64)),
    ("expanded row", lambda: _bf16(64).expand(24, 64), True, (False, False, 64)),
    ("weight row-slice, odd row stride", lambda: _bf16(96, 65)[:, :64], True, (False, False, 64)),
    ("neither dimension contiguous", lambda: _bf16(24, 128)[:, ::2], True, (False, False, 64)),
]


@pytest.mark.parametrize("make,mn_ok,want", [o[1:] for o in OPERANDS], ids=[o[0] for o in OPERANDS])
def test_gemm_operand_rule(make, mn_ok, want):
    t = make()
    g, mn, ld = ops._gemm_operand(t, mn_ok)
    assert ((g.data_ptr() == t.data_ptr() and g.stride() == t.stride()), mn, ld) == want
    assert torch.equal(g, t) and g.data_ptr() % 16 == 0


def test_linear_copies_the_views_the_library_would_refuse(lib):
    x, w = _unaligned(), _bf16(96, 72)[:, :64]
    y = ops.linear(x, w)
    ((name, A, W, bias, C, M, N, K, lda, ldw, ldc, act),) = lib.calls
    assert name == "lv_gemm_bias_act" and (M, N, K, lda, ldw, ldc) == (24, 96, 64, 64, 72, 96)
    assert A != x.data_ptr() and W == w.data_ptr() and C == y.data_ptr()
    lib.calls.clear()
    ops.linear(_bf16(4, 64), _bf16(96, 65)[:, :64])               # odd row stride: copied, not refused by the library
    assert lib.calls[0][9] == 64
