"""Restatements of the FP8 training quantisers (ops.quant_rows_fp8 with dtype=, ops.quant_cols_fp8_t) and CPU oracle
forms of the FP8 training operators, for tests/test_fp8_train_host.py and tests/test_gpu_fp8_train.py.

The rule (csrc/kv_fp8_core.h, with each format's largest finite value M: 448 for e4m3, 57 344 for e5m2), per row of
the row quantiser and per column of the cast-transpose: amax = max|x| in fp32; inv = M / amax (one IEEE division);
q = fp8_rn_satfinite(x * inv); scale = amax / M.  A row or column whose inv is not finite (amax 0, or a bf16-subnormal
amax below M / FLT_MAX) is zeros with scale 0.  The cast-transpose writes q [C, R16] with R16 = R rounded up to 16 and
zeros in columns R..R16.  torch's float32 -> float8 conversions round to nearest even; the clamp to +-M states the
satfinite saturation of the kernels' cvt.rn.satfinite.
"""
from __future__ import annotations

import contextlib

import torch

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FP8_MAX = {E4M3: 448.0, E5M2: 57344.0}


def quant_rows_ref(x: torch.Tensor, dtype=E4M3):
    """x [M, K] bf16 -> (q uint8 [M, K] in the bits of `dtype`, scale fp32 [M])."""
    mx = FP8_MAX[dtype]
    xf = x.float()
    amax = xf.abs().amax(-1, keepdim=True)
    inv = torch.full_like(amax, mx) / amax
    zero = torch.isinf(inv) | torch.isnan(inv)
    q = (xf * torch.where(zero, torch.zeros_like(inv), inv)).clamp(-mx, mx).to(dtype).view(torch.uint8)
    q = torch.where(zero, torch.zeros_like(q), q)
    scale = torch.where(zero, torch.zeros_like(amax), amax / mx)[..., 0]
    return q, scale


def quant_cols_t_ref(x: torch.Tensor, dtype=E4M3):
    """x [R, C] bf16 -> (q uint8 [C, R16], scale fp32 [C]): quant_rows_ref of x^T, padded with zero columns."""
    R = x.shape[0]
    q, scale = quant_rows_ref(x.t(), dtype)
    pad = -(-R // 16) * 16 - R
    return torch.cat([q, torch.zeros((q.shape[0], pad), dtype=torch.uint8)], dim=1), scale


def dequant(q: torch.Tensor, scale: torch.Tensor, dtype=None) -> torch.Tensor:
    """float64 q * scale[:, None]; q is an FP8 tensor, or uint8 bits of `dtype`."""
    if q.dtype == torch.uint8:
        q = q.view(dtype)
    return q.double() * scale.double()[:, None]


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
