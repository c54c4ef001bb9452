"""CPU oracle forms of the FP8 training operators (ops.quant_rows_fp8 with dtype=, ops.quant_cols_fp8_t,
ops.linear_fp8, ops._gemm_fp8_grad), for tests/test_fp8_train_host.py: the quantisers are the restatements of
tests/fp8_ref.py, the products float32 over the dequantised operands.
"""
from __future__ import annotations

import contextlib

import torch

from tests.fp8_ref import E4M3, quant_cols_t_ref, quant_rows_ref


# ------------------------------------------------------------------------------------------------
# CPU oracle forms of the FP8 operators (the host-logic harness, as tests/hostlogic.py does for the bf16 ones)
# ------------------------------------------------------------------------------------------------
def _quant_rows(x, dtype=E4M3):
    q, s = quant_rows_ref(x.contiguous(), dtype)
    return q.view(dtype), s


def _quant_cols_t(x, dtype=E4M3):
    q, s = quant_cols_t_ref(x.contiguous(), dtype)
    return q.view(dtype), s


def _linear_fp8(x, weight, bias=None, act=None, out=None):
    assert act in (None, "none") and out is None
    K = x.shape[-1]
    xq, xs = _quant_rows(x.reshape(-1, K))
    y = (xq.float() * xs[:, None]) @ weight.dequantize().t()
    if bias is not None:
        y = y + bias.float()
    return y.to(torch.bfloat16).view(*x.shape[:-1], -1)


def _gemm_fp8_grad(op, a, sa, b, sb, out, accumulate):
    r = (a.float() * sa[:, None]) @ (b.float() * sb[:, None]).t()
    if accumulate:
        out.add_(r)
    else:
        out.copy_(r.to(out.dtype))
    return out


FP8_SUBSTITUTES = {
    "quant_rows_fp8": _quant_rows,
    "quant_cols_fp8_t": _quant_cols_t,
    "linear_fp8": _linear_fp8,
    "_gemm_fp8_grad": _gemm_fp8_grad,
}


@contextlib.contextmanager
def oracle_fp8_ops():
    """tests.hostlogic.oracle_ops() plus the FP8 operators above."""
    from long_vita_b200 import ops
    from tests.hostlogic import oracle_ops

    saved = {name: getattr(ops, name) for name in FP8_SUBSTITUTES}
    try:
        with oracle_ops():
            for name, fn in FP8_SUBSTITUTES.items():
                setattr(ops, name, fn)
            yield ops
    finally:
        for name, fn in saved.items():
            setattr(ops, name, fn)
