"""The FP8 quantisation rule of csrc/fp8_core.h restated in torch, for every FP8 test, and the gcc build of that header.

The rule, per row of n values x, with M the largest finite value of the format (448 for e4m3, 57344 for e5m2):
amax = max|x| in fp32; inv = M / amax (one IEEE division); q = fp8_rn_satfinite(x * inv); scale = amax / M.  A row
whose inv is not finite (amax 0, or a bf16-subnormal amax below M / FLT_MAX) is zeros with scale 0.  torch's float32 ->
float8 conversions round to nearest even; the clamp to +-M states the satfinite saturation of the kernels'
cvt.rn.satfinite.  Both divisions are tensor by tensor: on CUDA a division by a Python scalar becomes a multiplication
by its reciprocal, so this restatement gives the same bits on any device.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np
import torch

from long_vita_b200 import ops

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FP8_MAX = {E4M3: 448.0, E5M2: 57344.0}
FMT = {E4M3: 0, E5M2: 1}                     # the `fmt` argument of csrc/fp8_core.h and the C entry points

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "long-vita_b200", "csrc")


def quant_rows_ref(x: torch.Tensor, dtype=E4M3):
    """x [..., n] bf16 -> (q [..., n] uint8 in the bits of `dtype`, scale [...] fp32), one scale per row."""
    xf = x.float()
    amax = xf.abs().amax(-1, keepdim=True)
    mx = torch.full_like(amax, FP8_MAX[dtype])
    inv = mx / amax
    zero = torch.isinf(inv) | torch.isnan(inv)
    q = (xf * torch.where(zero, torch.zeros_like(inv), inv)).clamp(-FP8_MAX[dtype], FP8_MAX[dtype])
    q = q.to(dtype).view(torch.uint8)
    q = torch.where(zero, torch.zeros_like(q), q)
    scale = torch.where(zero, torch.zeros_like(amax), amax / mx)[..., 0]
    return q, scale


def quant_cols_t_ref(x: torch.Tensor, dtype=E4M3):
    """Cast-transpose: x [R, C] bf16 -> (q uint8 [C, R16], scale fp32 [C]): quant_rows_ref of x^T, padded with zero
    columns to R16 = R rounded up to 16."""
    R = x.shape[0]
    q, scale = quant_rows_ref(x.t(), dtype)
    pad = -(-R // 16) * 16 - R
    return torch.cat([q, torch.zeros((q.shape[0], pad), dtype=torch.uint8, device=q.device)], dim=1), scale


def dequant(q: torch.Tensor, scale: torch.Tensor, dtype=None) -> torch.Tensor:
    """float64 q * scale[:, None]; q is an FP8 tensor, or uint8 bits of `dtype`."""
    if q.dtype == torch.uint8:
        q = q.view(dtype)
    return q.double() * scale.double()[:, None]


def finite_bf16() -> torch.Tensor:
    """Every finite bf16 value, both zeros included."""
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    return x[torch.isfinite(x.float())]


# ------------------------------------------------------------------------------------------------
# the FP8 host rows of the K/V cache: K heads, V heads, then the 2 hkv fp32 scales, zero-padded to 16 bytes
# ------------------------------------------------------------------------------------------------
def fp8_rows(k: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """k / v [n, hkv, d] bf16 -> the FP8 host rows uint8 [n, ops.kv_fp8_row_bytes(hkv, d)], each head one e4m3 row."""
    n, hkv, d = k.shape
    q, scale = quant_rows_ref(torch.cat([k, v], dim=1).cpu())
    pad = ops.kv_fp8_row_bytes(hkv, d) - 2 * hkv * d - 8 * hkv
    return torch.cat([q.reshape(n, -1), scale.contiguous().view(torch.uint8).reshape(n, -1),
                      torch.zeros(n, pad, dtype=torch.uint8)], dim=1)


def dequantise_rows(rows: torch.Tensor, hkv: int, d: int):
    """FP8 host rows -> (K, V) [n, hkv, d] fp32: float(q) * scale."""
    n = rows.shape[0]
    q = rows[:, : 2 * hkv * d].contiguous().view(E4M3).float().view(n, 2 * hkv, d)
    scale = rows[:, 2 * hkv * d : 2 * hkv * d + 8 * hkv].contiguous().view(torch.float32).view(n, 2 * hkv, 1)
    x = q * scale
    return x[:, :hkv], x[:, hkv:]


# ------------------------------------------------------------------------------------------------
# the headers built with gcc
# ------------------------------------------------------------------------------------------------
def build_shim(tmp_dir, source: str) -> ctypes.CDLL:
    """Compile `source` (C that includes csrc/fp8_core.h or csrc/attn_fp8_core.h) with gcc into a shared library in
    `tmp_dir` and load it.  No contraction and no fast-math, so each fp32 operation rounds as the kernels' does."""
    src, so = os.path.join(tmp_dir, "fp8_shim.c"), os.path.join(tmp_dir, "libfp8_shim.so")
    with open(src, "w") as f:
        f.write(source)
    subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-I", CSRC, src, "-o", so,
                    "-lm"], check=True)
    return ctypes.CDLL(so)


ROWS_SHIM = r"""
#include "fp8_core.h"
void quant_rows(int fmt, const uint16_t* x, uint8_t* q, float* scale, long long rows, long long n) {
  for (long long r = 0; r < rows; ++r) scale[r] = lv_fp8_quant_row(fmt, x + r * n, q + r * n, n);
}
long long kv8_row_bytes(long long hkv, long long d) { return lv_kv8_row_bytes(hkv, d); }
"""


def build_rows_shim(tmp_dir) -> ctypes.CDLL:
    """The row quantiser and the K/V host-row size of csrc/fp8_core.h (ROWS_SHIM), built with gcc."""
    lib = build_shim(tmp_dir, ROWS_SHIM)
    lib.quant_rows.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_longlong] * 2
    lib.kv8_row_bytes.restype = ctypes.c_longlong
    lib.kv8_row_bytes.argtypes = [ctypes.c_longlong, ctypes.c_longlong]
    return lib


def check_rows(lib, x: torch.Tensor, dtype=E4M3):
    """The header's row quantiser (build_rows_shim) over x [rows, n] bf16 -> (q uint8 [rows, n], scale fp32 [rows]),
    asserted byte for byte equal to quant_rows_ref."""
    x = x.contiguous()
    rows, n = x.shape
    q = np.zeros((rows, n), dtype=np.uint8)
    scale = np.zeros(rows, dtype=np.float32)
    lib.quant_rows(FMT[dtype], x.view(torch.int16).numpy().ctypes.data_as(ctypes.c_void_p),
                   q.ctypes.data_as(ctypes.c_void_p), scale.ctypes.data_as(ctypes.c_void_p), rows, n)
    q, scale = torch.from_numpy(q), torch.from_numpy(scale)
    q_ref, scale_ref = quant_rows_ref(x, dtype)
    bad = (q != q_ref).any(-1) | (scale.view(torch.int32) != scale_ref.view(torch.int32))
    assert not bool(bad.any()), (int(bad.sum()), x[bad][:4], q[bad][:4], q_ref[bad][:4])
    return q, scale
