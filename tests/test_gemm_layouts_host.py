"""The GEMM calls `ops.linear` makes for each operand layout, and the argument checks of `lv_gemm_ex`, on CPU.

`ops.linear` passes a 2-D transposed view (stride(0) == 1, stride(1) a multiple of 8, 16-byte aligned) to
`lv_gemm_ex` as an MN-major operand instead of copying it.  Contiguous operands keep making the `lv_gemm_bias_act`
call they made before `lv_gemm_ex` existed.  A stub library records the calls, so no GPU is needed.
"""
import types

import pytest
import torch

from long_vita_b200 import ops

E = 2       # bytes per bf16 element


class _Lib:
    def __init__(self):
        self.calls = []

    def lv_gemm_bias_act(self, A, W, bias, C, M, N, K, lda, ldw, ldc, act, stream):
        self.calls.append(("bias_act", A, W, bias, C, M, N, K, lda, ldw, ldc, act))
        return 0

    def lv_gemm_ex(self, A, W, bias, C, M, N, K, lda, ldw, ldc, a_mn, w_mn, act, stream):
        self.calls.append(("ex", A, W, bias, C, M, N, K, lda, ldw, ldc, a_mn, w_mn, act))
        return 0


@pytest.fixture
def lib(monkeypatch):
    fake = _Lib()
    monkeypatch.setattr(ops._lib, "lib", lambda: fake)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_need_cuda_bf16", lambda *ts: None)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
    return fake


def _bf16(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def test_contiguous_operands_make_the_same_bias_act_call(lib):
    x, w, b = _bf16(2, 5, 64), _bf16(96, 64), _bf16(96)
    y = ops.linear(x, w, b, act="gelu")
    assert y.shape == (2, 5, 96)
    (call,) = lib.calls
    assert call == ("bias_act", x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), 10, 96, 64, 64, 64, 96, 1)


def test_row_strided_x_is_read_in_place_by_bias_act(lib):
    buf = _bf16(10, 80)
    x = buf[:, :64]
    w = _bf16(96, 64)
    y = ops.linear(x, w)
    (call,) = lib.calls
    assert call == ("bias_act", x.data_ptr(), w.data_ptr(), None, y.data_ptr(), 10, 96, 64, 80, 64, 96, 0)


def test_transposed_x_is_mn_major(lib):
    xt = _bf16(64, 24)                  # stored [K, M]
    w = _bf16(96, 64)
    y = ops.linear(xt.t(), w)
    assert y.shape == (24, 96)
    (call,) = lib.calls
    assert call == ("ex", xt.data_ptr(), w.data_ptr(), None, y.data_ptr(), 24, 96, 64, 24, 64, 96, 1, 0, 0)


def test_transposed_weight_is_mn_major(lib):
    x = _bf16(10, 40)
    w = _bf16(40, 128)                  # nn.Linear weight [out = 40, in = 128]; dX = dY . W reads W^T
    y = ops.linear(x, w.t())
    assert y.shape == (10, 128)
    (call,) = lib.calls
    assert call == ("ex", x.data_ptr(), w.data_ptr(), None, y.data_ptr(), 10, 128, 40, 40, 128, 128, 0, 1, 0)


def test_both_transposed_with_an_odd_contraction_and_strided_storage(lib):
    dy = _bf16(13, 48)                  # [T, N], T = 13 tokens: no padding to a multiple of 8
    xs = _bf16(13, 72)                  # [T, 72] storage, X = its first 64 columns
    x = xs[:, :64]
    out = _bf16(48, 64)
    ops.linear(dy.t(), x.t(), out=out)
    (call,) = lib.calls
    assert call == ("ex", dy.data_ptr(), xs.data_ptr(), None, out.data_ptr(), 48, 64, 13, 48, 72, 64, 1, 1, 0)


def test_linear_wgrad_and_the_autograd_backward_read_transposed_views(lib, monkeypatch):
    T, n_in, n_out = 21, 64, 48
    x = _bf16(T, n_in).requires_grad_(True)
    w = _bf16(n_out, n_in).requires_grad_(True)
    y = ops.linear_autograd(x, w)
    lib.calls.clear()
    y.backward(_bf16(T, n_out))
    dx_call, dw_call = lib.calls
    assert dx_call[0] == "ex" and dx_call[2] == w.data_ptr() and dx_call[5:] == (T, n_in, n_out, n_out, n_in, n_in, 0, 1, 0)
    assert dw_call[0] == "ex" and dw_call[2] == x.data_ptr() and dw_call[5:] == (n_out, n_in, T, n_out, n_in, n_in, 1, 1, 0)


def test_views_the_kernel_cannot_read_are_copied_first(lib):
    # transposed, but the column stride is not a multiple of 8 elements
    xt = _bf16(64, 20)
    w = _bf16(96, 64)
    ops.linear(xt.t(), w)
    # transposed, but the first element is not 16-byte aligned
    st = _bf16(64, 40)
    xm = st[:, 1:25].t()
    assert xm.stride() == (1, 40) and xm.data_ptr() % 16 != 0
    ops.linear(xm, w)
    # neither dimension contiguous
    wx = _bf16(96, 128)[:, ::2]
    ops.linear(_bf16(10, 64), wx)
    assert [c[0] for c in lib.calls] == ["bias_act"] * 3
    for c in lib.calls:
        assert c[8] == 64 and c[9] == 64          # dense copies: lda = ldw = K
    assert lib.calls[0][1] != xt.data_ptr() and lib.calls[1][1] != st.data_ptr() + E


def test_lv_gemm_ex_rejects_bad_arguments_without_a_gpu(lib_built):
    from long_vita_b200 import _lib

    h = _lib.lib()

    def ex(*a):
        return h.lv_gemm_ex(*a, None), h.lv_last_error()

    P = 256          # a 16-byte aligned fake address: every case fails its checks before touching memory
    rc, msg = ex(None, P, None, P, 4, 8, 8, 8, 8, 8, 0, 0, 0)
    assert rc == -1 and b"null pointer" in msg
    rc, msg = ex(P, P, None, P, 4, 8, 8, 8, 8, 8, 2, 0, 0)
    assert rc == -1 and b"must be 0 or 1" in msg
    rc, msg = ex(P, P, None, P, 4, 8, 8, 8, 8, 8, 0, -1, 0)
    assert rc == -1 and b"must be 0 or 1" in msg
    rc, msg = ex(P, P, None, P, 4, 8, 7, 8, 8, 8, 1, 0, 0)      # K-major W needs K % 8 == 0
    assert rc == -1 and b"K=7" in msg
    rc, msg = ex(P, P, None, P, 4, 12, 8, 8, 16, 16, 1, 1, 0)
    assert rc == -1 and b"N=12" in msg
    rc, msg = ex(P, P, None, P, 20, 8, 7, 12, 8, 8, 1, 1, 0)    # MN-major A: lda a multiple of 8
    assert rc == -1 and b"lda=12" in msg
    rc, msg = ex(P, P, None, P, 20, 8, 7, 16, 8, 8, 1, 1, 0)    # ... and >= M
    assert rc == -1 and b"lda=16" in msg and b"M=20" in msg
    rc, msg = ex(P, P, None, P, 4, 64, 7, 8, 32, 64, 1, 1, 0)   # MN-major W: ldw >= N
    assert rc == -1 and b"ldw=32" in msg and b"N=64" in msg
    rc, msg = ex(P, P, None, P, 4, 64, 16, 8, 64, 60, 1, 1, 0)
    assert rc == -1 and b"ldc=60" in msg
    rc, msg = ex(P + 2, P, None, P, 4, 8, 7, 8, 8, 8, 1, 1, 0)
    assert rc == -1 and b"16-byte aligned" in msg
    rc, msg = ex(P, P, None, P, 4, 8, 7, 8, 8, 8, 1, 1, 5)
    assert rc == -1 and b"unknown activation" in msg
    rc, msg = ex(P, P, P, P, 4, 32, 7, 8, 32, 16, 1, 1, 3)
    assert rc == -1 and b"SwiGLU" in msg
    rc, msg = ex(P, P, None, P, 4, 8, 0, 8, 8, 8, 1, 1, 0)
    assert rc == -1 and b"bad shape" in msg


P16 = 256          # a 16-byte aligned fake address: every refused tuple fails its checks before touching memory
#                 A        W    bias  C    M   N   K   lda ldw ldc [a_mn w_mn] act
REFUSED = [
    ("lv_gemm_bias_act", (None, P16, None, P16, 4, 8, 8, 8, 8, 8, 0), [b"null pointer"]),
    ("lv_gemm_bias_act", (P16, P16, None, P16, -1, 8, 8, 8, 8, 8, 0), [b"bad shape"]),
    ("lv_gemm_bias_act", (P16, P16, None, P16, 4, 8, 0, 8, 8, 8, 0), [b"bad shape"]),
    ("lv_gemm_bias_act", (P16, P16, None, P16, 4, 8, 7, 8, 8, 8, 0), [b"K=7", b"multiples of 8"]),
    ("lv_gemm_bias_act", (P16, P16, None, P16, 4, 12, 8, 8, 8, 16, 0), [b"N=12", b"multiples of 8"]),
    ("lv_gemm_bias_act", (P16, P16, None, P16, 4, 8, 8, 8, 8, 8, 4), [b"unknown activation"]),
    ("lv_gemm_bias_act", (P16, P16, None, P16, 4, 8, 16, 8, 16, 8, 0), [b"lda=8", b"K=16"]),
    ("lv_gemm_bias_act", (P16, P16, None, P16, 4, 8, 16, 16, 12, 8, 0), [b"ldw=12"]),
    ("lv_gemm_bias_act", (P16, P16, None, P16, 4, 32, 16, 16, 16, 8, 0), [b"ldc=8"]),
    ("lv_gemm_bias_act", (P16, P16, P16, P16, 4, 32, 16, 16, 16, 16, 3), [b"SwiGLU"]),
    ("lv_gemm_ex", (P16, P16, None, P16, 4, 8, 8, 8, 8, 8, 0, 0, 0), []),         # K-major both: checked, then bias_act
    ("lv_gemm_ex", (P16 + 8, P16, None, P16, 4, 8, 8, 8, 8, 8, 0, 0, 0), [b"16-byte aligned"]),
    ("lv_gemm_ex", (P16, P16, None, P16, 4, 12, 8, 8, 8, 16, 0, 1, 0), [b"N=12"]),
    ("lv_gemm_ex", (P16, P16, None, P16, 4, 8, 8, 8, 4, 8, 0, 1, 0), [b"ldw=4", b"N=8"]),
    ("lv_gemm_ex", (P16, P16, None, P16, 4, 8, 1 << 31, 8, 8, 8, 1, 1, 0), [b"too large"]),
    ("lv_gemm_wgrad_acc_f32", (P16, P16, P16, 64, 64, 16, 64, 64, 64, 1, 1), []),   # accepted (stops at device binding)
    ("lv_gemm_wgrad_acc_f32", (P16, P16, P16, 64, 64, 16, 64, 64, 64, 1, 2), [b"must be 0 or 1"]),
    ("lv_gemm_wgrad_acc_f32", (P16, P16, P16, 64, 60, 16, 64, 64, 64, 1, 1), []),   # N a multiple of 4 is enough
    ("lv_gemm_wgrad_acc_f32", (P16, P16, P16, 64, 64, 7, 64, 64, 64, 1, 1), []),    # any K
]


@pytest.mark.parametrize("entry,args,msgs", REFUSED)
def test_gemm_entry_points_share_one_argument_check(lib_built, entry, args, msgs):
    """Refused tuples return -1 with the message; accepted ones pass the checks and stop at device binding here."""
    from long_vita_b200 import _lib

    h = _lib.lib()
    rc = getattr(h, entry)(*args, None)
    if msgs:
        assert rc == -1 and all(m in h.lv_last_error() for m in msgs), h.lv_last_error()
    else:
        assert rc != -1 or b"16-byte" in h.lv_last_error() or b"not device memory" in h.lv_last_error(), h.lv_last_error()
