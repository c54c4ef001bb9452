"""Operator layer: PyTorch tensors in / out, arithmetic in liblvb200.so through the C ABI.

PyTorch is used for device memory, streams and autograd plumbing only.  The C side cannot see tensor extents, so each
wrapper hands its tensors over as the kernel reads them - row matrices (`_rows`, `_like`), per-column parameters
(`_param`), index / label / statistics vectors (`_vec`), GEMM operands (`_gemm_operand`) - and a shape, length or dtype
mismatch raises ValueError naming the wrapper and the argument before anything is launched.  Tensors must be CUDA bf16
(or the stated integer / float type); RuntimeError is raised otherwise, when the extension is missing or when a call
fails - there is no eager fallback.
"""
from __future__ import annotations

import ctypes as C
import math
import weakref
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import AttnBwdParams, AttnDocs, AttnFp8Kv, AttnParams


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need_cuda_bf16(*ts: Optional[torch.Tensor]) -> None:
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("long_vita_b200 operators run on CUDA tensors only (no CPU fallback)")
        if t.dtype != torch.bfloat16:
            raise RuntimeError(f"expected bfloat16 tensor, got {t.dtype}")


def _need_cuda(t: torch.Tensor, dtype: torch.dtype) -> None:
    if not t.is_cuda or t.dtype != dtype:
        raise RuntimeError(f"expected CUDA {dtype} tensor, got {t.device} {t.dtype}")


def _call(name: str, *args) -> None:
    """Call the C entry point `name` with `args` and the current stream; RuntimeError if it fails."""
    _lib.check(getattr(_lib.lib(), name)(*args, _stream()), name)


def _rows(t: torch.Tensor, cols: int) -> torch.Tensor:
    """t [..., cols] as the contiguous row matrix [-1, cols] a kernel reads (copied only when it is not contiguous)."""
    return t.reshape(-1, cols).contiguous()


def _like(op: str, name: str, t: torch.Tensor, shape) -> torch.Tensor:
    """A companion operand (a residual, a gradient) as the contiguous [rows, cols] `shape` of the primary's rows."""
    if t.numel() != shape[0] * shape[1]:
        raise ValueError(f"{op}: {name} {tuple(t.shape)} does not hold the {shape[0]} rows of {shape[1]} it is read as")
    return (t if t.shape == shape else t.reshape(shape)).contiguous()


def _param(op: str, name: str, t: Optional[torch.Tensor], n: int) -> Optional[torch.Tensor]:
    """None, or t as the n contiguous elements a kernel reads (a per-column weight, bias or layer scale, a class token,
    a position table)."""
    if t is not None and t.numel() != n:
        raise ValueError(f"{op}: {name} {tuple(t.shape)} has {t.numel()} elements, the kernel reads {n}")
    return None if t is None else t.contiguous()


def _vec(op: str, name: str, t: torch.Tensor, dtype: torch.dtype, n: Optional[int] = None,
         inplace: bool = False) -> torch.Tensor:
    """An index, label or row-statistics tensor as the contiguous CUDA vector of `dtype` (and `n` elements, if given) a
    kernel reads; one the kernel writes (`inplace`) must already be contiguous."""
    if t.dtype != dtype or (n is not None and t.numel() != n) or (inplace and not t.is_contiguous()):
        want = f"{'a contiguous ' if inplace else ''}{dtype}{'' if n is None else f' of {n} elements'}"
        raise ValueError(f"{op}: {name} must be {want}, got {t.dtype} {tuple(t.shape)}")
    _need_cuda(t, dtype)
    return t.contiguous().view(-1)


class KernelTimer:
    """Optional per-launch device timing of the two tensor-core kernels (CUDA events on the
    launching stream).  bench.py installs one for its roofline numbers; None costs nothing."""

    def __init__(self):
        self.records = []  # (kind, algorithmic flops, start event, end event)

    def start(self):
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        return ev

    def stop(self, kind, flops, ev0):
        ev1 = torch.cuda.Event(enable_timing=True)
        ev1.record()
        self.records.append((kind, flops, ev0, ev1))

    def summary(self):
        """kind -> dict(launches, ms, flops); call after a synchronize."""
        out = {}
        for kind, flops, e0, e1 in self.records:
            d = out.setdefault(kind, {"launches": 0, "ms": 0.0, "flops": 0.0})
            d["launches"] += 1
            d["ms"] += e0.elapsed_time(e1)
            d["flops"] += flops
        return out


_TIMER: Optional[KernelTimer] = None


def set_kernel_timer(t: Optional[KernelTimer]) -> None:
    global _TIMER
    _TIMER = t


def launch_count() -> int:
    """Kernels launched by liblvb200.so so far in this process."""
    return int(_lib.lib().lv_launch_count())


# ------------------------------------------------------------------------------------------------
# packed documents (`--reset-position-ids --reset-attention-mask`)
# ------------------------------------------------------------------------------------------------
def _check_cu_host(cu, seq_len: Optional[int]) -> Tuple[int, ...]:
    cu = tuple(int(c) for c in cu)
    if len(cu) < 2 or cu[0] != 0 or any(b <= a for a, b in zip(cu, cu[1:])):
        raise ValueError(f"cu_seqlens must be 0 = c0 < c1 < ... < c_n (got {list(cu[:8])}{' ...' if len(cu) > 8 else ''})")
    if seq_len is not None and cu[-1] != seq_len:
        raise ValueError(f"cu_seqlens ends at {cu[-1]}, the packed row has {seq_len} tokens")
    if cu[-1] >= 2 ** 31:
        raise ValueError("cu_seqlens: sequence too long for int32 boundaries")
    return cu


def _mark_cu(cu_host: Tuple[int, ...], device) -> torch.Tensor:
    """int32 device tensor of validated boundaries; remembers the host copy so later calls neither sync nor re-check."""
    t = torch.tensor(cu_host, dtype=torch.int32, device=device)
    t._lv_cu_host = cu_host
    return t


def packed_cu_seqlens(position_ids: Optional[torch.Tensor] = None, actual_seq_len=None, *, device=None,
                      seq_len: Optional[int] = None) -> Optional[torch.Tensor]:
    """Document boundaries of one packed row, or None when the row holds a single sample.

    `actual_seq_len` is the reference's list of cumulative sample ends (long_vita/data/dataset_qwen2.py:160-166,
    published by training/utils.py:509-511): cu_seqlens = [0] + actual_seq_len.  From `position_ids` ([1, s], [s, 1] as
    Megatron stores them, or [s]) the boundaries are the rows after row 0 whose position is 0 - compute_actual_seq_len
    (training/utils.py:53-57), and transformers' prepare_fa_kwargs_from_position_ids for a row starting at 0.  A row
    whose positions never restart (including a zig-zag context-parallel shard, whose positions jump upwards) is not
    packed.  Returns a validated int32 tensor on `device` (default: that of position_ids, else the current CUDA
    device).  Call it once per forward: it reads the boundaries to the host (one synchronisation), the attention calls
    of every layer then reuse the tensor without another one.  Raises ValueError for micro-batch > 1, for packed
    position ids that do not start at 0, and for boundaries that are not strictly increasing or do not end at
    `seq_len`."""
    if (position_ids is None) == (actual_seq_len is None):
        raise ValueError("packed_cu_seqlens: pass exactly one of position_ids and actual_seq_len")
    if actual_seq_len is not None:
        ends = [int(e) for e in (actual_seq_len.reshape(-1).tolist() if torch.is_tensor(actual_seq_len) else actual_seq_len)]
        if len(ends) <= 1:
            if seq_len is not None and len(ends) == 1 and ends[0] != seq_len:
                raise ValueError(f"actual_seq_len ends at {ends[0]}, the packed row has {seq_len} tokens")
            return None
        cu = _check_cu_host([0] + ends, seq_len)
    else:
        pos = position_ids
        if pos.dim() == 2:
            if pos.shape[0] != 1 and pos.shape[1] != 1:
                raise ValueError(f"packed documents need micro-batch 1 (position_ids {tuple(pos.shape)})")
        elif pos.dim() != 1:
            raise ValueError(f"position_ids must be [1, s], [s, 1] or [s], got {tuple(pos.shape)}")
        flat = pos.reshape(-1).cpu()
        starts = (torch.nonzero(flat[1:] == 0).view(-1) + 1).tolist()
        if not starts:
            return None
        if int(flat[0]) != 0:
            raise ValueError(f"packed position_ids must start at 0 (got {int(flat[0])})")
        cu = _check_cu_host([0] + starts + [flat.numel()], seq_len)
        if device is None:
            device = pos.device
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return _mark_cu(cu, device)


def _docs_arg(cu_seqlens: torch.Tensor, seq_len: int):
    """(AttnDocs, host boundaries) of a cu_seqlens tensor; checked on the host unless packed_cu_seqlens made it."""
    _need_cuda(cu_seqlens, torch.int32)
    host = getattr(cu_seqlens, "_lv_cu_host", None)
    if host is None or host[-1] != seq_len or len(host) != cu_seqlens.numel():
        host = _check_cu_host(cu_seqlens.reshape(-1).tolist(), seq_len)
    elif not cu_seqlens.is_contiguous():
        raise ValueError("cu_seqlens must be contiguous")
    d = AttnDocs()
    d.cu_seqlens, d.n_docs = cu_seqlens.data_ptr(), len(host) - 1
    return d, host


def _docs_flops(host, hq: int, d: int) -> float:
    """Visible work of a packed row: 4 hq d sum_i L_i (L_i + 1) / 2."""
    return 4.0 * hq * d * sum((b - a) * (b - a + 1) / 2 for a, b in zip(host, host[1:]))


def docs_kwargs(cu_seqlens: Optional[torch.Tensor]) -> dict:
    """`cu_seqlens=` for the attention calls of a packed row, nothing for an unpacked one: unpacked calls keep exactly
    the arguments they had before document mode existed."""
    return {} if cu_seqlens is None else {"cu_seqlens": cu_seqlens}


def _check_docs_call(b, sq, sk, causal, q_seg_len, q_seg_pos, kv_pos0):
    if not causal:
        raise NotImplementedError("packed documents without a causal mask are not supported")
    if b != 1 or sq != sk:
        raise ValueError(f"packed documents need batch 1 and self-attention (got b={b}, sq={sq}, sk={sk})")
    if q_seg_len is not None or q_seg_pos is not None or kv_pos0:
        raise ValueError("packed documents take no q_seg_len / q_seg_pos / kv_pos0")


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def tma_view_ok(t: torch.Tensor) -> bool:
    """The attention kernels load q / k / v / out (and the gradients) through TMA, in place: the head dimension must be
    contiguous and every other stride a multiple of 8 elements (16 bytes)."""
    return t.stride(-1) == 1 and all(s % 8 == 0 for s in t.stride()[:-1])


def tma_view(t: torch.Tensor) -> torch.Tensor:
    return t if tma_view_ok(t) else t.contiguous()


def attn_params(q, k, v, out, lse=None, *, scale: Optional[float] = None, causal: bool, q_seg_len=None, q_seg_pos=None,
                kv_pos0: int = 0) -> AttnParams:
    """`lv_attn_params` of q [b, sq, hq, d], k / v [b, sk, hkv, d] and out [b, sq, hq, d] views (pointers and strides
    are taken as they are) and lse [b, hq, sq] fp32 or None.  Defaults: scale 1/sqrt(d), one query segment of sq rows
    whose mask is aligned to the last key (flash-attn >= 2.1)."""
    b, sq, hq, d = q.shape
    _, sk, hkv, _ = k.shape
    p = AttnParams()
    p.q, p.k, p.v, p.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    p.lse = _ptr(lse)
    p.batch, p.sq, p.sk, p.hq, p.hkv, p.d = b, sq, sk, hq, hkv, d
    for name, t in (("q_strides", q), ("k_strides", k), ("v_strides", v), ("o_strides", out)):
        arr = getattr(p, name)
        arr[0], arr[1], arr[2] = t.stride(0), t.stride(1), t.stride(2)
    p.scale = float(scale if scale is not None else 1.0 / math.sqrt(d))
    p.causal = 1 if causal else 0
    p.q_seg_len = int(q_seg_len if q_seg_len is not None else sq)
    if q_seg_pos is None:
        q_seg_pos = (sk - sq, 0)
    p.q_seg_pos[0], p.q_seg_pos[1] = int(q_seg_pos[0]), int(q_seg_pos[1])
    p.kv_pos0 = int(kv_pos0)
    return p


def attention_fwd(
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    *,
    causal: bool,
    scale: Optional[float] = None,
    layout: str = "bshd",
    return_lse: bool = False,
    q_seg_len: Optional[int] = None,
    q_seg_pos: Optional[Tuple[int, int]] = None,
    kv_pos0: int = 0,
    out: Optional[torch.Tensor] = None,
    cu_seqlens: Optional[torch.Tensor] = None,
):
    """softmax(scale * q k^T + mask) v.  `layout` names the dimension order of q/k/v and of the
    returned tensor: "bshd" (flash-attn / HF), "sbhd" (Megatron, dot_product_attention.py:344) or
    "bhsd" (HF AttentionInterface).  Strided views are consumed in place (no .contiguous()) as
    long as the head dimension is contiguous and the other strides are multiples of 8 elements.
    Returns out (same layout as q) or (out, lse[b, hq, sq] float32).

    `cu_seqlens` (int32 [n_docs + 1], see packed_cu_seqlens) makes the row a packed stream of documents: each query
    sees the keys of its own document up to itself (lv_attn_docs_fwd; batch 1, self-attention, causal only)."""
    _need_cuda_bf16(q, k, v)
    perm = {"bshd": (0, 1, 2, 3), "sbhd": (1, 0, 2, 3), "bhsd": (0, 2, 1, 3)}[layout]
    qv, kv_, vv = (t.permute(perm) for t in (q, k, v))  # views in b, s, h, d order
    b, sq, hq, d = qv.shape
    _, sk, hkv, _ = kv_.shape
    docs = host = None
    if cu_seqlens is not None:
        _check_docs_call(b, sq, sk, causal, q_seg_len, q_seg_pos, kv_pos0)
        docs, host = _docs_arg(cu_seqlens, sk)
    qv, kv_, vv = tma_view(qv), tma_view(kv_), tma_view(vv)
    if out is None:
        # allocate in the caller's layout so the result is contiguous there
        out = torch.empty(q.shape, dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((b, hq, sq), dtype=torch.float32, device=q.device) if return_lse else None
    p = attn_params(qv, kv_, vv, out.permute(perm), lse, scale=scale, causal=causal, q_seg_len=q_seg_len,
                    q_seg_pos=q_seg_pos, kv_pos0=kv_pos0)
    ev0 = _TIMER.start() if _TIMER is not None else None
    if docs is not None:
        _call("lv_attn_docs_fwd", C.byref(p), C.byref(docs))
    else:
        _call("lv_attn_fwd", C.byref(p))
    if ev0 is not None:
        if docs is not None:
            fl = _docs_flops(host, hq, d)
        elif causal and q_seg_len is None and sq == sk:
            fl = 4.0 * b * hq * d * (sq * (sq + 1) / 2)
        elif causal and q_seg_len is None and q_seg_pos is None and not kv_pos0 and sq < sk:
            # one query segment aligned to the last key (a query chunk over its key prefix): the visible pairs
            fl = 4.0 * b * hq * d * (sq * (sk - sq) + sq * (sq + 1) / 2)
        else:
            fl = 4.0 * b * hq * d * sq * sk  # upper bound for masked / segmented calls
        _TIMER.stop("attn_fwd", fl, ev0)
    return (out, lse) if return_lse else out


ATTN_FP8_BLOCK = 128   # key rows per K / V scale of the FP8 attention (csrc/attn_fp8_core.h)


def attn_fp8_kv_bytes(sk: int, hkv: int, d: int, batch: int = 1) -> int:
    """Device bytes of the quantised K / V that attention_fwd_fp8 holds during a call: K8 and Vt8 (e4m3, whole
    128-row blocks) and the two fp32 scales per block."""
    nt = -(-sk // ATTN_FP8_BLOCK)
    return batch * hkv * nt * (2 * ATTN_FP8_BLOCK * d + 8)


def attn_fp8_quant_kv(k: torch.Tensor, v: torch.Tensor):
    """K / V [b, sk, hkv, 128] bf16 views (strided, e.g. columns of a QKV buffer) -> (k8 [b, hkv, nt * 128, d],
    vt8 [b, hkv, nt, d, 128], k_scale, v_scale [b, hkv, nt]) in the layout of the FP8 attention (lv_attn_fp8_quant_kv;
    e4m3 as float8_e4m3fn, one scale per 128-key block, each V block transposed with the key permutation of
    csrc/attn_fp8_core.h)."""
    _need_cuda_bf16(k, v)
    if k.dim() != 4 or k.shape != v.shape:
        raise ValueError(f"attn_fp8_quant_kv: k {tuple(k.shape)} and v {tuple(v.shape)} must both be [b, sk, hkv, d]")
    kv_, vv = tma_view(k), tma_view(v)
    p = attn_params(kv_, kv_, vv, kv_, causal=True)
    return _attn_fp8_kv(p, k.device)[0]


def _attn_fp8_kv(p: AttnParams, device):
    """Quantise the K / V of the filled `p` (lv_attn_fp8_quant_kv) into new buffers; returns them and the AttnFp8Kv."""
    b, sk, hkv, d = p.batch, p.sk, p.hkv, p.d
    if d != 128:
        raise ValueError(f"FP8 attention: head_dim {d} is not supported (128 only)")
    nt = -(-sk // ATTN_FP8_BLOCK)
    k8 = torch.empty((b, hkv, nt * ATTN_FP8_BLOCK, d), dtype=torch.uint8, device=device)
    vt8 = torch.empty((b, hkv, nt, d, ATTN_FP8_BLOCK), dtype=torch.uint8, device=device)
    ks = torch.empty((b, hkv, nt), dtype=torch.float32, device=device)
    vs = torch.empty((b, hkv, nt), dtype=torch.float32, device=device)
    f = AttnFp8Kv()
    f.k8, f.vt8, f.k_scale, f.v_scale = k8.data_ptr(), vt8.data_ptr(), ks.data_ptr(), vs.data_ptr()
    _call("lv_attn_fp8_quant_kv", C.byref(p), C.byref(f))
    return (k8.view(FP8), vt8.view(FP8), ks, vs), f


def attention_fwd_fp8(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True,
                      return_lse: bool = False, *, scale: Optional[float] = None, out: Optional[torch.Tensor] = None):
    """Causal attention on the FP8 tensor cores (opt-in, lossy): q [b, sq, hq, 128], k / v [b, sk, hkv, 128] bf16
    ("bshd" views, consumed in place as attention_fwd consumes them), sq <= sk, the mask aligned to the last key.
    K and V are quantised into a temporary (attn_fp8_quant_kv, attn_fp8_kv_bytes), Q inside the kernel; the rule is
    that of csrc/attn_fp8_core.h.  Returns out [b, sq, hq, 128] bf16, or (out, lse [b, hq, sq] float32).  Anything
    else the FP8 kernel does not build (no causal mask, sq > sk, d != 128) is a ValueError before any launch; documents,
    query segments and context parallelism have no FP8 path."""
    _need_cuda_bf16(q, k, v)
    if not causal:
        raise ValueError("attention_fwd_fp8: only causal attention is built")
    if q.dim() != 4 or k.dim() != 4 or k.shape != v.shape:
        raise ValueError(f"attention_fwd_fp8: q {tuple(q.shape)}, k {tuple(k.shape)}, v {tuple(v.shape)} must be "
                         "[b, s, h, d] with k and v alike")
    b, sq, hq, d = q.shape
    sk = k.shape[1]
    if d != 128 or k.shape[0] != b or k.shape[3] != d or hq % k.shape[2] != 0:
        raise ValueError(f"attention_fwd_fp8: head_dim 128 and hq a multiple of hkv needed, got q {tuple(q.shape)}, "
                         f"k {tuple(k.shape)}")
    if sq > sk:
        raise ValueError(f"attention_fwd_fp8: sq={sq} > sk={sk} (the queries are the last sq rows of the keys)")
    qv, kv_, vv = tma_view(q), tma_view(k), tma_view(v)
    if out is None:
        out = torch.empty(q.shape, dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((b, hq, sq), dtype=torch.float32, device=q.device) if return_lse else None
    p = attn_params(qv, kv_, vv, out, lse, scale=scale, causal=True)
    ev0 = _TIMER.start() if _TIMER is not None else None
    bufs, f = _attn_fp8_kv(p, q.device)
    _call("lv_attn_fwd_fp8", C.byref(p), C.byref(f))
    del bufs                     # freed in stream order after the kernel
    if ev0 is not None:
        _TIMER.stop("attn_fwd_fp8", 4.0 * b * hq * d * (sq * (sk - sq) + sq * (sq + 1) / 2), ev0)
    return (out, lse) if return_lse else out


def attention_bwd(d_out, q, k, v, out, lse, *, causal: bool, scale: Optional[float] = None, q_seg_len=None,
                  q_seg_pos=None, kv_pos0: int = 0, cu_seqlens: Optional[torch.Tensor] = None,
                  dq: Optional[torch.Tensor] = None, dk: Optional[torch.Tensor] = None, dv: Optional[torch.Tensor] = None):
    """Gradients of attention_fwd (layout "bshd").  `out` / `lse` are the forward results, `cu_seqlens` the packed
    documents the forward was called with.  Returns (dq, dk, dv) with the shapes of q, k, v.  `dq` / `dk` / `dv`, all
    three or none, are caller buffers (strided views are fine, e.g. the per-head q / k / v columns of one dQKV buffer
    laid out like the fused QKV GEMM output) that the kernel writes through their strides."""
    if (dq is None) != (dk is None) or (dq is None) != (dv is None):
        raise ValueError("attention_bwd: pass all of dq, dk, dv or none")
    if dq is not None:
        _need_cuda_bf16(dq, dk, dv)
        for t, ref in ((dq, q), (dk, k), (dv, v)):
            if t.shape != ref.shape or not tma_view_ok(t):
                raise ValueError("attention_bwd: dq / dk / dv must have the shapes of q / k / v, a contiguous head dimension "
                                 "and strides that are multiples of 8 elements")
    _need_cuda_bf16(d_out, q, k, v, out)
    _need_cuda(lse, torch.float32)
    if tuple(lse.shape) != (q.shape[0], q.shape[2], q.shape[1]):
        raise ValueError(f"attention_bwd: lse {tuple(lse.shape)} is not [b, hq, sq] of q {tuple(q.shape)}")
    docs = None
    if cu_seqlens is not None:
        _check_docs_call(q.shape[0], q.shape[1], k.shape[1], causal, q_seg_len, q_seg_pos, kv_pos0)
        docs, _ = _docs_arg(cu_seqlens, k.shape[1])
    q, k, v, out, d_out = tma_view(q), tma_view(k), tma_view(v), tma_view(out), tma_view(d_out)
    if dq is None:
        dq, dk, dv = torch.empty_like(q, memory_format=torch.contiguous_format), \
            torch.empty_like(k, memory_format=torch.contiguous_format), torch.empty_like(v, memory_format=torch.contiguous_format)
    b, sq, hq, _ = q.shape
    delta = torch.empty((b, hq, sq), dtype=torch.float32, device=q.device)
    p = AttnBwdParams()
    p.fwd = attn_params(q, k, v, out, lse.contiguous(), scale=scale, causal=causal, q_seg_len=q_seg_len,
                        q_seg_pos=q_seg_pos, kv_pos0=kv_pos0)
    p.d_out, p.dq, p.dk, p.dv, p.delta_ws = d_out.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), delta.data_ptr()
    for name, t in (("do_strides", d_out), ("dq_strides", dq), ("dk_strides", dk), ("dv_strides", dv)):
        arr = getattr(p, name)
        arr[0], arr[1], arr[2] = t.stride(0), t.stride(1), t.stride(2)
    if docs is not None:
        _call("lv_attn_docs_bwd", C.byref(p), C.byref(docs))
    else:
        _call("lv_attn_bwd", C.byref(p))
    return dq, dk, dv


class _AttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, causal, scale, cu_seqlens):
        out, lse = attention_fwd(q, k, v, causal=causal, scale=scale, return_lse=True, **docs_kwargs(cu_seqlens))
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.causal, ctx.scale, ctx.cu_seqlens = causal, scale, cu_seqlens
        return out

    @staticmethod
    def backward(ctx, d_out):
        q, k, v, out, lse = ctx.saved_tensors
        dq, dk, dv = attention_bwd(d_out.contiguous(), q, k, v, out, lse, causal=ctx.causal, scale=ctx.scale,
                                   **docs_kwargs(ctx.cu_seqlens))
        return dq, dk, dv, None, None, None


def attention(q, k, v, *, causal: bool, scale: Optional[float] = None, cu_seqlens: Optional[torch.Tensor] = None):
    """Differentiable fused attention, "bshd" layout (the autograd twin of flash_attn_func; with `cu_seqlens`, of
    flash_attn_varlen_func over one packed row)."""
    return _AttentionFn.apply(q, k, v, causal, scale, cu_seqlens)


def _sm_count(device) -> int:
    return torch.cuda.get_device_properties(device).multi_processor_count if torch.cuda.is_available() else 132


def attention_decode(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, length: int, *,
                     scale: Optional[float] = None, n_splits: Optional[int] = None, return_lse: bool = False):
    """One new token against a K/V cache (SURVEY.md 8f-2; the reference has no such path - it re-prefills
    every generated token, long_vita_megatron/inference/text_generation/generation.py:127-135).

    q [hq, d]; k_cache / v_cache [>= length, hkv, d] (post-RoPE rows of the previous tokens, the new token's
    row already appended); returns out [hq, d] (and lse [hq] fp32, natural log - what a context-parallel
    combine across cache shards needs).

    HBM-bound (every K/V row is read once), so the job is to put all SMs on the cache: the G = hq / hkv query
    heads of a kv group become G query ROWS of one head (they share K/V), and the key range is cut into
    `n_splits` chunks that run as the batch dimension of the ordinary fused kernel (`lv_attn_fwd`,
    non-causal, with LSE); the partial results are merged by their log-sum-exp weights (flash-decoding).
    A ragged last chunk is a second launch with sk = remainder."""
    _need_cuda_bf16(q, k_cache, v_cache)
    hq, d = q.shape
    hkv = k_cache.shape[1]
    G = hq // hkv
    if length <= 0 or length > k_cache.shape[0]:
        raise ValueError(f"attention_decode: length {length} outside the cache (capacity {k_cache.shape[0]})")
    if n_splits is None:
        n_splits = max(1, _sm_count(q.device) // hkv)
    per = -(-length // n_splits)
    chunk = max(128, (per + 127) // 128 * 128)                             # keys per split, whole 128-key tiles
    n_full, rem = divmod(length, chunk)
    qp = q.view(hkv, G, d).transpose(0, 1)                                 # [G rows, hkv heads, d]
    outs, lses = [], []
    if n_full:
        qb = qp.unsqueeze(0).expand(n_full, G, hkv, d).contiguous()
        kb = k_cache[: n_full * chunk].view(n_full, chunk, hkv, d)
        vb = v_cache[: n_full * chunk].view(n_full, chunk, hkv, d)
        o, l = attention_fwd(qb, kb, vb, causal=False, scale=scale, return_lse=True)   # [n, G, hkv, d], [n, hkv, G]
        outs.append(o)
        lses.append(l)
    if rem:
        o, l = attention_fwd(qp.unsqueeze(0).contiguous(), k_cache[n_full * chunk : length].unsqueeze(0),
                             v_cache[n_full * chunk : length].unsqueeze(0), causal=False, scale=scale, return_lse=True)
        outs.append(o)
        lses.append(l)
    o = outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)              # [n, G, hkv, d]
    l = lses[0] if len(lses) == 1 else torch.cat(lses, dim=0)              # [n, hkv, G]
    return decode_merge(o, l, return_lse=return_lse)


def decode_merge(o_part: torch.Tensor, lse_part: torch.Tensor, return_lse: bool = False):
    """o_part [n, G, hkv, d] bf16, lse_part [n, hkv, G] fp32 -> out [hq, d] (head h = kvh * G + g) and the
    merged log-sum-exp [hq]: out = sum_s exp(lse_s - LSE) o_s (lv_attn_decode_merge)."""
    _need_cuda_bf16(o_part)
    n, G, hkv, d = o_part.shape
    o_part, lse_part = o_part.contiguous(), _vec("decode_merge", "lse_part", lse_part, torch.float32, n * hkv * G)
    out = torch.empty((hkv * G, d), dtype=torch.bfloat16, device=o_part.device)
    lse = torch.empty((hkv * G,), dtype=torch.float32, device=o_part.device) if return_lse else None
    _call("lv_attn_decode_merge", o_part.data_ptr(), lse_part.data_ptr(), out.data_ptr(), _ptr(lse), n, G, hkv, d)
    return (out, lse) if return_lse else out


# ------------------------------------------------------------------------------------------------
# K/V rows in pinned host memory (the host tier of kv_cache.OffloadedKVCache)
# ------------------------------------------------------------------------------------------------
def _is_pinned(t: torch.Tensor) -> bool:
    return not t.is_cuda and t.is_pinned()


def _host_rows(op: str, name: str, t: torch.Tensor, cols: Optional[int] = None,
               dtype: torch.dtype = torch.bfloat16) -> None:
    """t must be a pinned host row matrix [rows, cols] of `dtype` with contiguous rows (the kernel reads it by
    address)."""
    if not _is_pinned(t):
        raise ValueError(f"{op}: {name} must be pinned host memory, got {t.device}"
                         f"{'' if t.is_cuda else ' (not pinned)'}")
    if t.dtype != dtype or t.dim() != 2 or (cols is not None and t.shape[1] != cols) \
            or t.stride() != (t.shape[1], 1):
        want = "[rows, cols]" if cols is None else f"[rows, {cols}]"
        raise ValueError(f"{op}: {name} must be a contiguous {str(dtype).replace('torch.', '')} {want}, got "
                         f"{t.dtype} {tuple(t.shape)} strides {t.stride()}")


def pinned_rows(rows: int, cols: int, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """An uninitialised [rows, cols] tensor of `dtype` in pinned, device-mapped host memory of exactly that size
    (lv_host_alloc; a caching pinned allocator rounds a buffer up to a power of two).  The memory is released when
    the last tensor viewing it is gone."""
    n = int(rows) * int(cols) * torch.empty((), dtype=dtype).element_size()
    p = C.c_void_p()
    _lib.check(_lib.lib().lv_host_alloc(n, C.byref(p)), "lv_host_alloc")
    buf = (C.c_uint8 * n).from_address(p.value)
    weakref.finalize(buf, _lib.lib().lv_host_free, p.value).atexit = False     # the process exit releases it
    return torch.frombuffer(buf, dtype=dtype).view(rows, cols)


def kv_fp8_row_bytes(hkv: int, d: int) -> int:
    """Bytes of one FP8 host row (csrc/fp8_core.h): K and V of the hkv heads in e4m3, then the 2 hkv fp32 scales
    padded to 16 bytes; 2112 at 8 kv heads of 128."""
    return 2 * hkv * d + (8 * hkv + 15) // 16 * 16


def pinned_fp8_rows(rows: int, hkv: int, d: int) -> torch.Tensor:
    """The uninitialised uint8 [rows, kv_fp8_row_bytes(hkv, d)] rows of an FP8 host layer (pinned_rows)."""
    return pinned_rows(rows, kv_fp8_row_bytes(hkv, d), torch.uint8)


def _kv_source(op: str, k: torch.Tensor, v: torch.Tensor, dst: torch.Tensor) -> int:
    """Row stride (elements) of the device K/V rows k / v [n, hkv, d] that V follows K in; dst must have n rows."""
    n, hkv, d = k.shape
    rs = k.stride(0) if n > 1 else 2 * hkv * d          # a single row's stride is arbitrary
    if (v.shape != k.shape or not (k[0].is_contiguous() and v[0].is_contiguous()) or (n > 1 and v.stride(0) != rs)
            or rs % 8 or rs < 2 * hkv * d or v.data_ptr() != k.data_ptr() + hkv * d * k.element_size()):
        raise ValueError(f"{op}: k / v {tuple(k.shape)} strides {k.stride()} / {v.stride()} are not the "
                         f"K and V halves of one row")
    if dst.shape[0] != n:
        raise ValueError(f"{op}: dst has {dst.shape[0]} rows for {n}")
    return rs


def kv_rows_to_host(k: torch.Tensor, v: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
    """Copy the K/V rows k / v [n, hkv, d] (device views whose V follows K in each row, as in the QKV GEMM output or
    the streamed layer's K|V buffer) into the host rows dst [n, 2 hkv d] (pinned; row = K heads | V heads), in stream
    order and without a device temporary: one strided copy (lv_rows_to_host).  Returns dst."""
    _need_cuda_bf16(k, v)
    n, hkv, d = k.shape
    _host_rows("kv_rows_to_host", "dst", dst, 2 * hkv * d)
    rs = _kv_source("kv_rows_to_host", k, v, dst)
    _call("lv_rows_to_host", dst.data_ptr(), k.data_ptr(), n, 2 * hkv * d * 2, rs * 2)
    return dst


def kv_rows_to_host_fp8(k: torch.Tensor, v: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
    """kv_rows_to_host into FP8 host rows: dst uint8 [n, kv_fp8_row_bytes(hkv, d)] (pinned) receives the rows of k / v
    [n, hkv, d] quantised per head (csrc/fp8_core.h), in stream order, by a kernel that stores straight into the
    mapped host rows (lv_rows_to_host_fp8; no device temporary).  d = 128.  Returns dst."""
    _need_cuda_bf16(k, v)
    n, hkv, d = k.shape
    _host_rows("kv_rows_to_host_fp8", "dst", dst, kv_fp8_row_bytes(hkv, d), torch.uint8)
    rs = _kv_source("kv_rows_to_host_fp8", k, v, dst)
    _call("lv_rows_to_host_fp8", dst.data_ptr(), k.data_ptr(), n, hkv, d, rs * 2)
    return dst


def attention_decode_host(q: torch.Tensor, kv_host: torch.Tensor, length: int, *, scale: Optional[float] = None,
                          n_splits: Optional[int] = None, return_lse: bool = False):
    """attention_decode over K/V rows in pinned host memory: q [hq, d] (d = 128) on the device, kv_host
    [capacity, 2 hkv d] bf16 pinned (row = K of the hkv heads | V of the hkv heads, post-RoPE, the new token's row
    already written); rows [0, length) are read in place over PCIe by lv_attn_decode_host, split into `n_splits`
    contiguous key ranges (default: one per SM), and merged by lv_attn_decode_merge.  Returns out [hq, d] (and lse
    [hq] fp32, natural log)."""
    _need_cuda_bf16(q)
    if q.dim() != 2:
        raise ValueError(f"attention_decode_host: q must be [hq, d], got {tuple(q.shape)}")
    hq, d = q.shape
    _host_rows("attention_decode_host", "kv_host", kv_host)
    cap, cols = kv_host.shape
    hkv = cols // (2 * d)
    if hkv == 0 or cols != 2 * hkv * d or hq % hkv:
        raise ValueError(f"attention_decode_host: kv_host rows of {cols} are not K|V of kv heads of {d} for {hq} "
                         f"query heads")
    if not 0 < length <= cap:
        raise ValueError(f"attention_decode_host: length {length} outside the cache (capacity {cap})")
    if n_splits is None:
        n_splits = max(1, min(_sm_count(q.device), -(-length // 128)))
    G = hq // hkv
    o = torch.empty((n_splits, G, hkv, d), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((n_splits, hkv, G), dtype=torch.float32, device=q.device)
    _call("lv_attn_decode_host", q.contiguous().data_ptr(), kv_host.data_ptr(), o.data_ptr(), lse.data_ptr(), length,
          cap, hq, hkv, d, n_splits, float(scale if scale is not None else 1.0 / math.sqrt(d)))
    return decode_merge(o, lse, return_lse=return_lse)


def attention_decode_host_fp8(q: torch.Tensor, kv_host: torch.Tensor, length: int, *, scale: Optional[float] = None,
                              n_splits: Optional[int] = None, return_lse: bool = False):
    """attention_decode_host over FP8 host rows: kv_host uint8 [capacity, kv_fp8_row_bytes(hkv, d)] pinned (written by
    kv_rows_to_host_fp8), read in place by lv_attn_decode_host_fp8 with the same split rule and merged by
    lv_attn_decode_merge.  The result is attention over the dequantised rows, not over the bf16 ones.  Returns out
    [hq, d] (and lse [hq] fp32, natural log)."""
    _need_cuda_bf16(q)
    if q.dim() != 2:
        raise ValueError(f"attention_decode_host_fp8: q must be [hq, d], got {tuple(q.shape)}")
    hq, d = q.shape
    _host_rows("attention_decode_host_fp8", "kv_host", kv_host, dtype=torch.uint8)
    cap, cols = kv_host.shape
    hkv = cols // (2 * d + 8)                            # kv_fp8_row_bytes(h, d) is in [h (2d + 8), h (2d + 8) + 8)
    if hkv == 0 or cols != kv_fp8_row_bytes(hkv, d) or hq % hkv:
        raise ValueError(f"attention_decode_host_fp8: kv_host rows of {cols} bytes are not FP8 K|V rows of kv heads "
                         f"of {d} for {hq} query heads")
    if not 0 < length <= cap:
        raise ValueError(f"attention_decode_host_fp8: length {length} outside the cache (capacity {cap})")
    if n_splits is None:
        n_splits = max(1, min(_sm_count(q.device), -(-length // 128)))
    G = hq // hkv
    o = torch.empty((n_splits, G, hkv, d), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((n_splits, hkv, G), dtype=torch.float32, device=q.device)
    _call("lv_attn_decode_host_fp8", q.contiguous().data_ptr(), kv_host.data_ptr(), o.data_ptr(), lse.data_ptr(),
          length, cap, hq, hkv, d, n_splits, float(scale if scale is not None else 1.0 / math.sqrt(d)))
    return decode_merge(o, lse, return_lse=return_lse)


def merge_attention(o_part: torch.Tensor, lse_part: torch.Tensor, return_lse: bool = False):
    """The attention of M query rows over the union of n disjoint key sets, from its n parts: o_part [n, M, hq, d] bf16
    and lse_part [n, hq, M] fp32 (natural log; attention_fwd's lse without the batch) -> out [M, hq, d] (and lse
    [hq, M]).  lv_attn_decode_merge with the M hq rows as the query heads of one kv head (G = M hq, hkv = 1), so
    M hq < 2^20."""
    n, M, hq, d = o_part.shape
    if M * hq >= 1 << 20:
        raise ValueError(f"merge_attention: {M} query rows of {hq} heads exceed the merge's 2^20 rows")
    out, lse = decode_merge(o_part.reshape(n, M * hq, 1, d), lse_part.transpose(1, 2).reshape(n, 1, M * hq),
                            return_lse=True)
    out = out.view(M, hq, d)
    return (out, lse.view(M, hq).t().contiguous()) if return_lse else out


def kv_rows_dequant_fp8(src: torch.Tensor, hkv: int, d: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """FP8 host rows copied to the device, src uint8 [n, kv_fp8_row_bytes(hkv, d)], -> bf16 K|V rows [n, 2 hkv d]
    (written to `out` if given), each value bf16_rn(float(q) * scale) (csrc/fp8_core.h; lv_kv_rows_dequant_fp8)."""
    _need_cuda(src, torch.uint8)
    if src.dim() != 2 or src.shape[1] != kv_fp8_row_bytes(hkv, d) or not src.is_contiguous():
        raise ValueError(f"kv_rows_dequant_fp8: src must be contiguous FP8 rows [n, {kv_fp8_row_bytes(hkv, d)}], got "
                         f"{tuple(src.shape)}")
    n = src.shape[0]
    if out is None:
        out = torch.empty((n, 2 * hkv * d), dtype=torch.bfloat16, device=src.device)
    _need_cuda_bf16(out)
    if tuple(out.shape) != (n, 2 * hkv * d) or not out.is_contiguous():
        raise ValueError(f"kv_rows_dequant_fp8: out must be a contiguous [{n}, {2 * hkv * d}], got {tuple(out.shape)}")
    _call("lv_kv_rows_dequant_fp8", src.data_ptr(), out.data_ptr(), n, hkv, d)
    return out


def _copy_to_device(dst: torch.Tensor, src: torch.Tensor) -> None:
    """dst.copy_(src) from pinned host rows, asynchronously on the current stream (the copy engine)."""
    dst.copy_(src, non_blocking=True)


HOST_ROWS_CHUNK = 65536
HOST_ROWS_PARTS_BYTES = 1 << 30       # chunk results held at once by attention_host_rows before a merge


def attention_host_rows(q: torch.Tensor, kv_host: torch.Tensor, length: int, *, chunk_rows: int = HOST_ROWS_CHUNK,
                        return_lse: bool = False):
    """M >= 1 query rows q [M, hq, d] (device) attend, unmasked, to the rows [0, length) of a host layer of the K/V
    cache: kv_host pinned, bf16 [capacity, 2 hkv d] or FP8 uint8 [capacity, kv_fp8_row_bytes(hkv, d)].  Returns out
    [M, hq, d] (and lse [hq, M] fp32, natural log).

    The rows are not read in place: the copy engine stages them, `chunk_rows` at a time, into a ring of two device
    buffers on a side stream, while the current stream runs the previous chunk; an FP8 chunk is copied as FP8 and
    decoded to bf16 in HBM (kv_rows_dequant_fp8).  Each chunk is one attention_fwd over K / V views of the staged rows,
    the ragged last one a shorter call, and the chunk results are merged by merge_attention.  So every host row
    crosses PCIe once, whatever M is.  Stream order: the side stream first waits for the work enqueued before the
    call (the rows may have just been written to the host), a buffer is refilled only after the call that read it, and
    the current stream waits for each copy before it reads the buffer.  Refused with ValueError before anything is
    launched: rows that are not pinned or not of the layer's width, length outside [1, capacity], a chunk_rows that is
    not a positive multiple of 128, M hq >= 2^20.

    The chunk results are held until they are merged: when all n of them would take more than HOST_ROWS_PARTS_BYTES
    (many small chunks for many query rows), they are merged in groups of about sqrt(n) and the group results once
    more, so that at most ~2 sqrt(n) of them exist at a time."""
    _need_cuda_bf16(q)
    op = "attention_host_rows"
    if q.dim() != 3:
        raise ValueError(f"{op}: q must be [M, hq, d], got {tuple(q.shape)}")
    M, hq, d = q.shape
    fp8 = kv_host.dtype == torch.uint8
    _host_rows(op, "kv_host", kv_host, dtype=torch.uint8 if fp8 else torch.bfloat16)
    cap, cols = kv_host.shape
    hkv = cols // (2 * d + 8) if fp8 else cols // (2 * d)
    if hkv == 0 or cols != (kv_fp8_row_bytes(hkv, d) if fp8 else 2 * hkv * d) or hq % hkv:
        raise ValueError(f"{op}: kv_host rows of {cols} {'bytes' if fp8 else 'values'} are not "
                         f"{'FP8 ' if fp8 else ''}K|V rows of kv heads of {d} for {hq} query heads")
    if not 0 < length <= cap:
        raise ValueError(f"{op}: length {length} outside the cache (capacity {cap})")
    if chunk_rows <= 0 or chunk_rows % 128:
        raise ValueError(f"{op}: chunk_rows {chunk_rows} is not a positive multiple of 128")
    if M * hq >= 1 << 20:
        raise ValueError(f"{op}: {M} query rows of {hq} heads exceed the merge's 2^20 rows")
    n = -(-length // chunk_rows)
    rows = min(chunk_rows, length)
    group = n if n * M * hq * d * 2 <= HOST_ROWS_PARTS_BYTES else math.isqrt(n - 1) + 1
    dev = q.device
    cur = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(device=dev)
    stage = [torch.empty((rows, cols), dtype=kv_host.dtype, device=dev) for _ in range(2)]
    kv = torch.empty((rows, 2 * hkv * d), dtype=torch.bfloat16, device=dev) if fp8 else None
    o_part = torch.empty((group, M, hq, d), dtype=torch.bfloat16, device=dev)
    lse_part = torch.empty((group, hq, M), dtype=torch.float32, device=dev)
    groups = -(-n // group)
    o_grp = torch.empty((groups, M, hq, d), dtype=torch.bfloat16, device=dev) if groups > 1 else None
    lse_grp = torch.empty((groups, hq, M), dtype=torch.float32, device=dev) if groups > 1 else None
    q4 = q.unsqueeze(0)

    def after(stream):
        ev = torch.cuda.Event()
        ev.record(stream)
        return ev

    side.wait_event(after(cur))
    ready, free = [None, None], [None, None]

    def fill(i):
        b, r0 = i % 2, i * chunk_rows
        r1 = min(r0 + chunk_rows, length)
        if free[b] is not None:
            side.wait_event(free[b])
        with torch.cuda.stream(side):
            _copy_to_device(stage[b][: r1 - r0], kv_host[r0:r1])
        ready[b] = after(side)

    fill(0)
    for i in range(n):
        if i + 1 < n:
            fill(i + 1)
        b, r = i % 2, min(chunk_rows, length - i * chunk_rows)
        cur.wait_event(ready[b])
        rows_i = stage[b][:r]
        if fp8:
            rows_i = kv_rows_dequant_fp8(rows_i, hkv, d, out=kv[:r])
            free[b] = after(cur)
        k = rows_i[:, : hkv * d].view(r, hkv, d).unsqueeze(0)
        v = rows_i[:, hkv * d :].view(r, hkv, d).unsqueeze(0)
        j = i % group
        _, lse = attention_fwd(q4, k, v, causal=False, return_lse=True, out=o_part[j : j + 1])
        lse_part[j].copy_(lse[0])
        if not fp8:
            free[b] = after(cur)
        if groups > 1 and (j == group - 1 or i == n - 1):
            o, lse = merge_attention(o_part[: j + 1], lse_part[: j + 1], return_lse=True)
            o_grp[i // group].copy_(o)
            lse_grp[i // group].copy_(lse)
    if groups > 1:
        return merge_attention(o_grp, lse_grp, return_lse=return_lse)
    return merge_attention(o_part, lse_part, return_lse=return_lse)


# ------------------------------------------------------------------------------------------------
# token-wise operators
# ------------------------------------------------------------------------------------------------
def _out_rows(op: str, out: torch.Tensor, shape, *inputs: torch.Tensor) -> torch.Tensor:
    """A caller's output buffer as the contiguous [rows, cols] `shape` the kernel writes.  It may be one of `inputs`
    itself (in place: each of these kernels writes an element only from the thread that read it, after reading it)
    but must not partly overlap one, where a thread would overwrite rows another thread has still to read."""
    _need_cuda_bf16(out)
    if out.numel() != shape[0] * shape[1] or not out.is_contiguous():
        raise ValueError(f"{op}: out {tuple(out.shape)} must be a contiguous tensor of the {shape[0]} rows of {shape[1]} "
                         "it receives")
    lo, hi = out.data_ptr(), out.data_ptr() + 2 * out.numel()
    for t in inputs:
        if t is not None and t.data_ptr() != lo and t.data_ptr() < hi and lo < t.data_ptr() + 2 * t.numel():
            raise ValueError(f"{op}: out overlaps an input without being it")
    return out.view(shape)


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, residual: Optional[torch.Tensor] = None,
            out: Optional[torch.Tensor] = None):
    """RMSNorm over the last dim.  With `residual`, returns (norm(x + residual), x + residual); `out`, if given,
    receives x + residual (it may be `residual` or `x` itself, e.g. a row slice of the residual stream)."""
    _need_cuda_bf16(x, weight, residual)
    cols = x.shape[-1]
    x2 = _rows(x, cols)
    res2 = None if residual is None else _like("rmsnorm", "residual", residual, x2.shape)
    if out is not None and residual is None:
        raise ValueError("rmsnorm: out receives x + residual; it needs a residual")
    weight = _param("rmsnorm", "weight", weight, cols)
    y = torch.empty_like(x2)
    if residual is None:
        s = None
    else:
        s = torch.empty_like(x2) if out is None else _out_rows("rmsnorm", out, x2.shape, x2, res2)
    _call("lv_rmsnorm", x2.data_ptr(), _ptr(res2), weight.data_ptr(), y.data_ptr(), _ptr(s), x2.shape[0], cols, float(eps))
    if s is None:
        return y.view(x.shape)
    return y.view(x.shape), (s.view(x.shape) if out is None else out)


def layernorm(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], eps: float = 1e-6):
    _need_cuda_bf16(x, weight, bias)
    cols = x.shape[-1]
    x2 = _rows(x, cols)
    weight, bias = _param("layernorm", "weight", weight, cols), _param("layernorm", "bias", bias, cols)
    y = torch.empty_like(x2)
    _call("lv_layernorm", x2.data_ptr(), weight.data_ptr(), _ptr(bias), y.data_ptr(), x2.shape[0], cols, float(eps))
    return y.view(x.shape)


def rope_table(pos: torch.Tensor, inv_freq: torch.Tensor):
    """cos, sin tables (bf16 [n, 2 * len(inv_freq)]) for int64 positions `pos` [n]."""
    pos, inv_freq = _vec("rope_table", "pos", pos, torch.int64), _vec("rope_table", "inv_freq", inv_freq, torch.float32)
    dim = 2 * inv_freq.numel()
    cos = torch.empty((pos.numel(), dim), dtype=torch.bfloat16, device=pos.device)
    sin = torch.empty_like(cos)
    _call("lv_rope_table", pos.data_ptr(), inv_freq.data_ptr(), cos.data_ptr(), sin.data_ptr(), pos.numel(), dim)
    return cos, sin


def rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, out: Optional[torch.Tensor] = None):
    """Rotate-half RoPE of x[n_tok, heads, dim] (a strided view is fine) with cos / sin [n_tok, dim]; returns a new
    tensor or writes `out` (which may be x itself)."""
    _need_cuda_bf16(x, cos, sin)
    if x.dim() != 3 or x.stride(2) != 1:
        raise ValueError(f"rope: x {tuple(x.shape)} must be [n_tok, heads, dim] with a contiguous last dimension")
    n_tok, heads, dim = x.shape
    cos, sin = _like("rope", "cos", cos, (n_tok, dim)), _like("rope", "sin", sin, (n_tok, dim))
    if out is None:
        out = torch.empty((n_tok, heads, dim), dtype=torch.bfloat16, device=x.device)
    elif out.shape != x.shape or out.stride(2) != 1:
        raise ValueError(f"rope: out {tuple(out.shape)} must have x's shape and a contiguous last dimension")
    _call("lv_rope", x.data_ptr(), out.data_ptr(), cos.data_ptr(), sin.data_ptr(), n_tok, heads, dim, x.stride(0),
          x.stride(1), out.stride(0), out.stride(1))
    return out


def swiglu(gate_up: torch.Tensor):
    _need_cuda_bf16(gate_up)
    inter = gate_up.shape[-1] // 2
    g2 = _rows(gate_up, 2 * inter)
    out = torch.empty((g2.shape[0], inter), dtype=torch.bfloat16, device=gate_up.device)
    _call("lv_swiglu", g2.data_ptr(), out.data_ptr(), g2.shape[0], inter)
    return out.view(*gate_up.shape[:-1], inter)


def bias_gelu(x: torch.Tensor, bias: Optional[torch.Tensor] = None, approximate: str = "none"):
    _need_cuda_bf16(x, bias)
    cols = x.shape[-1]
    x2 = _rows(x, cols)
    bias = _param("bias_gelu", "bias", bias, cols)
    y = torch.empty_like(x2)
    _call("lv_bias_gelu", x2.data_ptr(), _ptr(bias), y.data_ptr(), x2.shape[0], cols, 1 if approximate == "tanh" else 0)
    return y.view(x.shape)


def ls_residual(x: torch.Tensor, y: torch.Tensor, ls: Optional[torch.Tensor] = None,
                bias: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None):
    """x + (y + bias) * ls (layer-scale residual); ls / bias optional.  `out`, if given, receives the result (it may
    be `x` or `y` itself: `ls_residual(x, d, out=x)` is x += d)."""
    _need_cuda_bf16(x, y, ls, bias)
    cols = x.shape[-1]
    x2 = _rows(x, cols)
    y2 = _like("ls_residual", "y", y, x2.shape)
    ls, bias = _param("ls_residual", "ls", ls, cols), _param("ls_residual", "bias", bias, cols)
    o2 = torch.empty_like(x2) if out is None else _out_rows("ls_residual", out, x2.shape, x2, y2)
    _call("lv_ls_residual", x2.data_ptr(), y2.data_ptr(), _ptr(bias), _ptr(ls), o2.data_ptr(), x2.shape[0], cols)
    return o2.view(x.shape) if out is None else out


def pixel_shuffle(x: torch.Tensor, hw: int, has_cls: bool):
    """[n, (1 +) hw*hw, c] -> [n, (hw/2)^2, 4c]."""
    _need_cuda_bf16(x)
    if x.dim() != 3 or x.shape[1] != hw * hw + (1 if has_cls else 0):
        raise ValueError(f"pixel_shuffle: x {tuple(x.shape)} is not [n, (1 +) {hw}*{hw}, c]")
    x = x.contiguous()
    n, _, c = x.shape
    out = torch.empty((n, (hw // 2) ** 2, 4 * c), dtype=torch.bfloat16, device=x.device)
    _call("lv_pixel_shuffle", x.data_ptr(), out.data_ptr(), n, hw, c, 1 if has_cls else 0)
    return out


def embed_scatter(ids: torch.Tensor, table: torch.Tensor, feat: Optional[torch.Tensor] = None,
                  dst_idx: Optional[torch.Tensor] = None, src_idx: Optional[torch.Tensor] = None):
    """out[t] = table[ids[t]]; out[dst_idx[i]] = feat[src_idx[i]] (src_idx None => i)."""
    _need_cuda_bf16(table, feat)
    ids = _vec("embed_scatter", "ids", ids, torch.int64)
    n_tok, hidden = ids.numel(), table.shape[1]
    out = torch.empty((n_tok, hidden), dtype=torch.bfloat16, device=table.device)
    n_sc = 0
    if feat is not None:
        feat = _rows(feat, hidden)
        dst_idx = _vec("embed_scatter", "dst_idx", dst_idx, torch.int64)
        n_sc = dst_idx.numel()
        if src_idx is not None:
            src_idx = _vec("embed_scatter", "src_idx", src_idx, torch.int64, n_sc)
    _call("lv_embed_scatter", ids.data_ptr(), table.data_ptr(), table.shape[0], _ptr(feat), _ptr(src_idx), _ptr(dst_idx),
          n_sc, out.data_ptr(), n_tok, hidden)
    return out


def row_gather(x: torch.Tensor, idx: torch.Tensor):
    _need_cuda_bf16(x)
    x = x.contiguous()
    idx = _vec("row_gather", "idx", idx, torch.int64)
    out = torch.empty((idx.numel(), x.shape[1]), dtype=torch.bfloat16, device=x.device)
    _call("lv_row_gather", x.data_ptr(), idx.data_ptr(), out.data_ptr(), idx.numel(), x.shape[1])
    return out


def row_scatter_zero(x: torch.Tensor, idx: torch.Tensor, n_rows_out: int):
    _need_cuda_bf16(x)
    x = x.contiguous()
    idx = _vec("row_scatter_zero", "idx", idx, torch.int64)
    out = torch.empty((n_rows_out, x.shape[1]), dtype=torch.bfloat16, device=x.device)
    _call("lv_row_scatter_zero", x.data_ptr(), idx.data_ptr(), out.data_ptr(), idx.numel(), n_rows_out, x.shape[1])
    return out


def row_scatter(x: torch.Tensor, idx: torch.Tensor, out: torch.Tensor):
    """out[idx[i]] = x[i] in place, every other row of out untouched: x [n, cols], idx n int64 row indices, out a
    contiguous [rows, cols].  Returns out."""
    _need_cuda_bf16(x, out)
    if out.dim() != 2 or not out.is_contiguous():
        raise ValueError(f"row_scatter: out {tuple(out.shape)} must be a contiguous row matrix")
    x = _rows(x, out.shape[1])
    idx = _vec("row_scatter", "idx", idx, torch.int64, x.shape[0])
    _call("lv_row_scatter", x.data_ptr(), idx.data_ptr(), out.data_ptr(), idx.numel(), out.shape[0], out.shape[1])
    return out


# ------------------------------------------------------------------------------------------------
# dense linears
# ------------------------------------------------------------------------------------------------
_ACT = {None: 0, "none": 0, "gelu": 1, "gelu_tanh": 2, "swiglu": 3}


def _gemm_operand(t: torch.Tensor, mn_ok: bool = True) -> Tuple[torch.Tensor, bool, int]:
    """How the wgmma GEMM reads the 2-D operand t [rows, K]: (tensor, mn_major, leading dimension).  K-major in place
    when K is contiguous, the row stride a multiple of 8 elements and >= K (no overlapping rows) and the start 16-byte
    aligned; else, unless mn_ok is False, MN-major in place under the same conditions with the two dimensions swapped
    (t.t() of such a [K, rows] tensor); else a contiguous K-major copy."""
    (rows, K), (s0, s1) = t.shape, t.stride()
    aligned = t.data_ptr() % 16 == 0
    if s1 == 1 and s0 % 8 == 0 and s0 >= K and aligned:
        return t, False, s0
    if mn_ok and s0 == 1 and s1 % 8 == 0 and s1 >= rows and aligned:
        return t, True, s1
    t = t.clone(memory_format=torch.contiguous_format)
    return t, False, t.stride(0)


def linear(x: torch.Tensor, weight, bias: Optional[torch.Tensor] = None, act: Optional[str] = None,
           out: Optional[torch.Tensor] = None):
    """act(x @ weight.T + bias); weight is [N, K] (nn.Linear layout).  Either operand may also be a 2-D transposed
    view (stride(0) == 1, stride(1) a multiple of 8, e.g. t.t() of a contiguous [K, X]): the kernel reads it in place
    (lv_gemm_ex) instead of a contiguous copy.  Any other layout is copied to a contiguous tensor first.  An Fp8Weight
    runs the FP8 product instead (linear_fp8)."""
    if isinstance(weight, Fp8Weight):
        return linear_fp8(x, weight, bias, act, out)
    _need_cuda_bf16(x, weight, bias)
    K = x.shape[-1]
    if weight.dim() != 2 or weight.shape[1] != K:
        raise ValueError(f"linear: weight {tuple(weight.shape)} is not [N, K={K}]")
    N = weight.shape[0]
    bias = _param("linear", "bias", bias, N)
    x2, a_mn, lda = _gemm_operand(x.reshape(-1, K))
    weight, w_mn, ldw = _gemm_operand(weight)
    M = x2.shape[0]
    n_out = N // 2 if act == "swiglu" else N      # fused SwiGLU: weight rows interleaved (gate_i, up_i)
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.bfloat16, device=x.device)
    if M == 0:      # e.g. a context-parallel rank that owns no answer token (empty logit mask)
        return out.view(*x.shape[:-1], n_out)
    ev0 = _TIMER.start() if _TIMER is not None else None
    if a_mn or w_mn:
        _call("lv_gemm_ex", x2.data_ptr(), weight.data_ptr(), _ptr(bias), out.data_ptr(), M, N, K, lda, ldw, out.stride(0),
              int(a_mn), int(w_mn), _ACT[act])
    else:       # the entry point whose decode-sized GEMV path also takes an unaligned `out`
        _call("lv_gemm_bias_act", x2.data_ptr(), weight.data_ptr(), _ptr(bias), out.data_ptr(), M, N, K, lda, ldw,
              out.stride(0), _ACT[act])
    if ev0 is not None:
        _TIMER.stop("gemm_bf16", 2.0 * M * N * K, ev0)
    return out.view(*x.shape[:-1], n_out)


# ------------------------------------------------------------------------------------------------
# FP8 (e4m3) linears: per-row scales on both operands (csrc/fp8_core.h), lv_gemm_fp8
# ------------------------------------------------------------------------------------------------
FP8 = torch.float8_e4m3fn
FP8_E5M2 = torch.float8_e5m2
_FP8_FMT = {FP8: 0, FP8_E5M2: 1}            # the `fmt` argument of the C entry points


def _fp8_fmt(op: str, dtype) -> int:
    if dtype not in _FP8_FMT:
        raise ValueError(f"{op}: dtype must be torch.float8_e4m3fn or torch.float8_e5m2, got {dtype!r}")
    return _FP8_FMT[dtype]


def quant_rows_fp8(x: torch.Tensor, dtype: torch.dtype = FP8) -> Tuple[torch.Tensor, torch.Tensor]:
    """x bf16 [M, K] (K contiguous, K a multiple of 16, row stride a multiple of 8) -> (q [M, K] of `dtype`, scale
    fp32 [M]): one scale per row, amax / max, q = fp8(x * max / amax) saturating at max, the largest finite value of
    `dtype` (e4m3, the default, or e5m2); a row of zeros (or too small to scale) is zeros with scale 0
    (lv_quant_rows_fp8_fmt, the rule of csrc/fp8_core.h).  x ~ q.float() * scale[:, None]."""
    _need_cuda_bf16(x)
    fmt = _fp8_fmt("quant_rows_fp8", dtype)
    if x.dim() != 2:
        raise ValueError(f"quant_rows_fp8: x must be [M, K], got {tuple(x.shape)}")
    M, K = x.shape
    if K == 0 or K % 16:
        raise ValueError(f"quant_rows_fp8: K={K} must be a positive multiple of 16")
    if x.stride(1) != 1 or x.stride(0) % 8 or x.data_ptr() % 16:
        x = x.contiguous()
    q = torch.empty((M, K), dtype=dtype, device=x.device)
    scale = torch.empty((M,), dtype=torch.float32, device=x.device)
    if M:
        _call("lv_quant_rows_fp8_fmt", x.data_ptr(), q.data_ptr(), scale.data_ptr(), M, K, max(x.stride(0), K), fmt)
    return q, scale


def quant_cols_fp8_t(x: torch.Tensor, dtype: torch.dtype = FP8) -> Tuple[torch.Tensor, torch.Tensor]:
    """Cast-transpose: x bf16 [R, C] (C contiguous, C a multiple of 8, row stride a multiple of 8) -> (q [C, R16] of
    `dtype`, scale fp32 [C]) with q[c, r] = x[r, c] quantised by the scale of column c (the rule of quant_rows_fp8
    applied to each column) and R16 = R rounded up to 16, columns R..R16 of q being zero, so that q is a K-major
    operand of the FP8 GEMM with the R rows of x as its contraction (lv_quant_cols_fp8_t).
    x ~ (q.float() * scale[:, None]).t()[:R]."""
    _need_cuda_bf16(x)
    fmt = _fp8_fmt("quant_cols_fp8_t", dtype)
    if x.dim() != 2:
        raise ValueError(f"quant_cols_fp8_t: x must be [R, C], got {tuple(x.shape)}")
    R, Cn = x.shape
    if Cn == 0 or Cn % 8:
        raise ValueError(f"quant_cols_fp8_t: C={Cn} must be a positive multiple of 8")
    if x.stride(1) != 1 or (R > 1 and x.stride(0) % 8) or x.data_ptr() % 16:
        x = x.contiguous()
    q = torch.empty((Cn, -(-R // 16) * 16), dtype=dtype, device=x.device)
    scale = torch.empty((Cn,), dtype=torch.float32, device=x.device)
    amax_ws = torch.empty((Cn,), dtype=torch.int32, device=x.device)
    _call("lv_quant_cols_fp8_t", x.data_ptr(), q.data_ptr(), scale.data_ptr(), amax_ws.data_ptr(), R, Cn,
          x.stride(0) if R > 1 else Cn, fmt)
    return q, scale


class Fp8Weight:
    """A linear layer's weight in FP8: data e4m3 [N, K] with one fp32 scale per output channel (row), scale [N]; the
    weight reads back as data.float() * scale[:, None].  Row slicing w[a:b] slices both (the Q and K|V rows of a fused
    QKV weight).  ops.linear takes it in place of a bf16 weight."""

    __slots__ = ("data", "scale")

    def __init__(self, data: torch.Tensor, scale: torch.Tensor):
        if data.dtype != FP8 or data.dim() != 2 or scale.dtype != torch.float32 or scale.shape != (data.shape[0],):
            raise ValueError(f"Fp8Weight: data must be float8_e4m3fn [N, K] and scale float32 [N], got {data.dtype} "
                             f"{tuple(data.shape)} and {scale.dtype} {tuple(scale.shape)}")
        self.data, self.scale = data, scale

    @classmethod
    def quantize(cls, w: torch.Tensor) -> "Fp8Weight":
        """The bf16 weight w [N, K] quantised per row (quant_rows_fp8)."""
        return cls(*quant_rows_fp8(w))

    @property
    def shape(self) -> torch.Size:
        return self.data.shape

    @property
    def device(self) -> torch.device:
        return self.data.device

    def dim(self) -> int:
        return 2

    def nbytes(self) -> int:
        return self.data.numel() + 4 * self.scale.numel()

    def __getitem__(self, rows) -> "Fp8Weight":
        if not isinstance(rows, slice) or rows.step not in (None, 1):
            raise TypeError("Fp8Weight: only contiguous row slices w[a:b] are supported")
        return Fp8Weight(self.data[rows], self.scale[rows])

    def to(self, device) -> "Fp8Weight":
        return Fp8Weight(self.data.to(device), self.scale.to(device))

    def dequantize(self) -> torch.Tensor:
        """The fp32 weight it stands for."""
        return self.data.float() * self.scale[:, None]


def linear_fp8(x: torch.Tensor, weight: Fp8Weight, bias: Optional[torch.Tensor] = None, act: Optional[str] = None,
               out: Optional[torch.Tensor] = None):
    """act(bf16((x_q @ w_q.T) * s_x * s_w + bias)): x bf16 [..., K] is quantised per row (quant_rows_fp8), then
    lv_gemm_fp8 multiplies it with the FP8 weight [N, K] (a GEMV for up to 4 rows).  act is None or "swiglu" (weight
    rows interleaved (gate_i, up_i), no bias).  `out`, if given, is a bf16 [M, N or N / 2] row matrix with
    contiguous rows, 16-byte aligned, whose row stride is a multiple of 8 (e.g. rows of a wider buffer)."""
    for name, t, dtype in (("x", x, torch.bfloat16), ("bias", bias, torch.bfloat16), ("out", out, torch.bfloat16),
                           ("weight.data", weight.data, FP8), ("weight.scale", weight.scale, torch.float32)):
        if t is not None and t.dtype != dtype:
            raise ValueError(f"linear_fp8: {name} must be {dtype}, got {t.dtype}")
    _need_cuda_bf16(x, bias)
    _need_cuda(weight.data, FP8)
    _need_cuda(weight.scale, torch.float32)
    K = x.shape[-1]
    N = weight.shape[0]
    if weight.shape[1] != K:
        raise ValueError(f"linear_fp8: weight {tuple(weight.shape)} is not [N, K={K}]")
    if K % 16:
        raise ValueError(f"linear_fp8: K={K} must be a multiple of 16")
    if act not in (None, "none", "swiglu"):
        raise ValueError(f"linear_fp8: activation {act!r} is not built (None or 'swiglu')")
    if N % (16 if act == "swiglu" else 8):
        raise ValueError(f"linear_fp8: N={N} must be a multiple of {16 if act == 'swiglu' else 8}")
    if act == "swiglu" and bias is not None:
        raise ValueError("linear_fp8: the fused SwiGLU takes no bias")
    if weight.data.stride(1) != 1 or weight.data.stride(0) % 16 or weight.data.data_ptr() % 16:
        raise ValueError(f"linear_fp8: weight rows must be contiguous and 16-byte aligned with a row stride that is a "
                         f"multiple of 16, got strides {weight.data.stride()}")
    bias = _param("linear_fp8", "bias", bias, N)
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    n_out = N // 2 if act == "swiglu" else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.bfloat16, device=x.device)
    else:
        _need_cuda_bf16(out)
        if (out.dim() != 2 or out.shape != (M, n_out) or out.stride(1) != 1
                or (M > 1 and (out.stride(0) % 8 or out.stride(0) < n_out)) or out.data_ptr() % 16):
            raise ValueError(f"linear_fp8: out {tuple(out.shape)} strides {out.stride()} is not a 16-byte aligned "
                             f"[{M}, {n_out}] row matrix with a row stride that is a multiple of 8")
    if M == 0:
        return out.view(*x.shape[:-1], n_out)
    if x2.stride(1) != 1 or x2.stride(0) % 8 or x2.data_ptr() % 16:
        x2 = x2.contiguous()
    # the quantised A operand in one temporary, e4m3 rows then their fp32 scales: a decode step is bound by host work
    # per launch, so the FP8 call allocates once more than the bf16 one, not twice
    ws = torch.empty((M * K + 4 * M,), dtype=torch.uint8, device=x.device)
    xq, xs = ws.data_ptr(), ws.data_ptr() + M * K
    _call("lv_quant_rows_fp8_fmt", x2.data_ptr(), xq, xs, M, K, max(x2.stride(0), K), _FP8_FMT[FP8])
    ev0 = _TIMER.start() if _TIMER is not None else None
    ldc = out.stride(0) if M > 1 else -(-n_out // 8) * 8
    _call("lv_gemm_fp8", xq, xs, weight.data.data_ptr(), weight.scale.data_ptr(), _ptr(bias),
          out.data_ptr(), M, N, K, K, weight.data.stride(0), ldc, _ACT[act])
    if ev0 is not None:
        _TIMER.stop("gemm_fp8", 2.0 * M * N * K, ev0)
    return out.view(*x.shape[:-1], n_out)


# ------------------------------------------------------------------------------------------------
# FP8 training of a linear: backward products on lv_gemm_fp8_grad.  Both operands of every product are K-major with
# one scale per row (FP8 wgmma reads nothing else), so each backward operand is an FP8 copy quantised along the axis
# the product reduces over:
#   forward  Y  [T, N] = X [T, K] . W [N, K]^T      X per token (row),      W per output channel (row)
#   dgrad    dX [T, K] = dY [T, N] . (W^T) [K, N]^T  dY per token (row),     W^T per input channel (quant_cols_fp8_t)
#   wgrad    dW [N, K] = (dY^T) [N, T] . (X^T) [K, T]^T   dY^T per output channel, X^T per input channel
#                                                        (both quant_cols_fp8_t, T padded to 16 with zeros)
# ------------------------------------------------------------------------------------------------
def _gemm_fp8_grad(op: str, a: torch.Tensor, sa: torch.Tensor, b: torch.Tensor, sb: torch.Tensor, out: torch.Tensor,
                   accumulate: bool) -> torch.Tensor:
    """out [M, N] (bf16; fp32 added into with `accumulate`) from A [M, K] (e4m3 / e5m2) and B [N, K] (e4m3), both
    K-major with 16-byte aligned rows (lv_gemm_fp8_grad)."""
    (M, K), N = a.shape, b.shape[0]
    if b.dtype != FP8 or a.dtype not in _FP8_FMT or b.shape[1] != K or sa.shape != (M,) or sb.shape != (N,):
        raise ValueError(f"{op}: operands {a.dtype} {tuple(a.shape)} and {b.dtype} {tuple(b.shape)} (scales "
                         f"{tuple(sa.shape)}, {tuple(sb.shape)}) are not FP8 [M, K], e4m3 [N, K] with one scale per row")
    for t in (a, b):
        if t.stride(1) != 1 or (t.shape[0] > 1 and t.stride(0) % 16) or t.data_ptr() % 16:
            raise ValueError(f"{op}: FP8 operand strides {t.stride()} are not 16-byte aligned rows")
    if M == 0:
        return out
    ev0 = _TIMER.start() if _TIMER is not None else None
    _call("lv_gemm_fp8_grad", a.data_ptr(), _FP8_FMT[a.dtype], sa.data_ptr(), b.data_ptr(), sb.data_ptr(),
          out.data_ptr(), M, N, K, a.stride(0) if M > 1 else K, b.stride(0) if N > 1 else K, out.stride(0),
          int(accumulate))
    if ev0 is not None:
        _TIMER.stop("gemm_fp8", 2.0 * M * N * K, ev0)
    return out


def linear_fp8_dgrad(dy: torch.Tensor, weight_t: "Fp8Weight", dtype: torch.dtype = FP8) -> torch.Tensor:
    """dX [..., K] = dY [..., N] . W [N, K] in FP8: dY bf16 quantised per token in `dtype` (quant_rows_fp8), weight_t
    = Fp8Weight(*quant_cols_fp8_t(W)), the e4m3 [K, N] copy of W scaled per input channel.  N a multiple of 16.
    Returns bf16."""
    _need_cuda_bf16(dy)
    N = dy.shape[-1]
    if N % 16 or weight_t.shape[1] != N:
        raise ValueError(f"linear_fp8_dgrad: dY [..., {N}] and W^T {tuple(weight_t.shape)} are not [.., N], [K, N] "
                         "with N a multiple of 16")
    dq, ds = quant_rows_fp8(dy.reshape(-1, N), dtype)
    dx = torch.empty((dq.shape[0], weight_t.shape[0]), dtype=torch.bfloat16, device=dy.device)
    _gemm_fp8_grad("linear_fp8_dgrad", dq, ds, weight_t.data, weight_t.scale, dx, False)
    return dx.view(*dy.shape[:-1], weight_t.shape[0])


def _wgrad_operands(op: str, dy2: torch.Tensor, x_t, dtype):
    _need_cuda_bf16(dy2)
    T, N = dy2.shape
    xq, xs = x_t
    if xq.dim() != 2 or xq.shape[1] != -(-T // 16) * 16:
        raise ValueError(f"{op}: X^T {tuple(xq.shape)} is not the [K, {-(-T // 16) * 16}] cast-transpose of {T} tokens")
    dq, ds = quant_cols_fp8_t(dy2, dtype)
    return dq, ds, xq, xs


def linear_fp8_wgrad(dy2: torch.Tensor, x_t: Tuple[torch.Tensor, torch.Tensor],
                     dtype: torch.dtype = FP8) -> torch.Tensor:
    """dW [N, K] = dY^T [N, T] . X [T, K] in FP8, the token dimension T being the contraction: dY bf16 [T, N] is
    cast-transposed in `dtype` (quant_cols_fp8_t), x_t = quant_cols_fp8_t(X) (e4m3 [K, T16], scale [K]) is X^T.
    Without tokens dW is zero and nothing is launched.  Returns bf16."""
    T, N = dy2.shape
    if T == 0:
        return torch.zeros((N, x_t[0].shape[0]), dtype=torch.bfloat16, device=dy2.device)
    dq, ds, xq, xs = _wgrad_operands("linear_fp8_wgrad", dy2, x_t, dtype)
    dw = torch.empty((N, xq.shape[0]), dtype=torch.bfloat16, device=dy2.device)
    return _gemm_fp8_grad("linear_fp8_wgrad", dq, ds, xq, xs, dw, False)


def linear_fp8_wgrad_accumulate(dy2: torch.Tensor, x_t: Tuple[torch.Tensor, torch.Tensor], main_grad: torch.Tensor,
                                dtype: torch.dtype = FP8) -> torch.Tensor:
    """main_grad [N, K] fp32 += the product of linear_fp8_wgrad, in place: each element gets one fp32 add of the value
    whose bf16 rounding linear_fp8_wgrad returns.  main_grad: unit column stride, a row stride that is a multiple of 4,
    16-byte aligned (as linear_wgrad_accumulate).  Without tokens nothing is launched.  Returns main_grad."""
    _need_cuda(main_grad, torch.float32)
    T, N = dy2.shape
    if tuple(main_grad.shape) != (N, x_t[0].shape[0]):
        raise RuntimeError(f"linear_fp8_wgrad_accumulate: main_grad is {tuple(main_grad.shape)}, the weight gradient "
                           f"is [{N}, {x_t[0].shape[0]}]")
    if main_grad.stride(1) != 1 or main_grad.stride(0) % 4 != 0 or main_grad.data_ptr() % 16 != 0:
        raise RuntimeError(f"linear_fp8_wgrad_accumulate: main_grad (strides {main_grad.stride()}) must have unit "
                           "column stride, a row stride that is a multiple of 4 and a 16-byte aligned start")
    if T == 0:
        return main_grad
    dq, ds, xq, xs = _wgrad_operands("linear_fp8_wgrad_accumulate", dy2, x_t, dtype)
    return _gemm_fp8_grad("linear_fp8_wgrad_accumulate", dq, ds, xq, xs, main_grad, True)


class _LinearFp8Fn(torch.autograd.Function):
    """y = x W^T + b in FP8 (linear_fp8 on W quantised per output channel), with the backward of _LinearFn in FP8: dX
    by linear_fp8_dgrad on W^T quantised per input channel, dW by linear_fp8_wgrad[_accumulate], gradients quantised
    in `grad_dtype`.  Both copies of W are made from the weight as it is when they are needed - W in the forward, W^T
    in the backward - so whatever writes the weight between steps (an optimizer copying into .data included) is seen,
    and no FP8 weight copy outlives its product.  The forward keeps only X^T in e4m3 with its scales for dW (one byte
    per element), or, without fp8_wgrad, X in bf16 for the bf16 wgrad."""

    @staticmethod
    def forward(ctx, x, weight, bias, grad_dtype, fp8_wgrad, accumulate_wgrad):
        K = x.shape[-1]
        ctx.grad_dtype, ctx.fp8_wgrad = grad_dtype, fp8_wgrad
        ctx.has_bias, ctx.accumulate_wgrad, ctx.x_shape = bias is not None, accumulate_wgrad, x.shape
        ctx.weight = weight
        if not ctx.needs_input_grad[1]:
            ctx.save_for_backward()
        elif fp8_wgrad:
            ctx.save_for_backward(*quant_cols_fp8_t(x.reshape(-1, K)))
        else:
            ctx.save_for_backward(x)
        return linear_fp8(x, Fp8Weight.quantize(weight.detach()), bias)

    @staticmethod
    def backward(ctx, dy):
        weight = ctx.weight
        n_out, k_in = weight.shape
        dy2 = dy.reshape(-1, n_out).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            w_t = Fp8Weight(*quant_cols_fp8_t(weight.detach()))
            dx = linear_fp8_dgrad(dy2, w_t, ctx.grad_dtype).view(ctx.x_shape)
        if ctx.needs_input_grad[1]:
            saved = ctx.saved_tensors
            main_grad = fused_wgrad_main_grad(weight) if ctx.accumulate_wgrad else None
            if ctx.fp8_wgrad:
                if main_grad is None:
                    dw = linear_fp8_wgrad(dy2, saved, ctx.grad_dtype)
                else:
                    linear_fp8_wgrad_accumulate(dy2, saved, main_grad, ctx.grad_dtype)
            else:
                x2 = saved[0].reshape(-1, k_in)
                if main_grad is None:
                    dw = linear_wgrad(dy2, x2)
                else:
                    linear_wgrad_accumulate(dy2, x2, main_grad)
            if main_grad is not None:
                dw = fused_wgrad_dummy(weight, main_grad, dy2.dtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.float().sum(dim=0).to(dy2.dtype)
        return dx, dw, db, None, None, None


def linear_fp8_autograd(x, weight, bias=None, grad_dtype: torch.dtype = FP8, fp8_wgrad: bool = True,
                        accumulate_wgrad: bool = False):
    """Differentiable FP8 linear (see _LinearFp8Fn): weight is the bf16 parameter [N, K] (N a multiple of 16: dgrad's
    contraction) that receives the gradient.  Scales are current scales, computed from the tensor being quantised.
    accumulate_wgrad: as linear_autograd."""
    _fp8_fmt("linear_fp8_autograd", grad_dtype)
    if weight.dim() != 2 or weight.shape[0] % 16:
        raise ValueError(f"linear_fp8_autograd: weight {tuple(weight.shape)} must be [N, K] with N a multiple of 16")
    return _LinearFp8Fn.apply(x, weight, bias, grad_dtype, bool(fp8_wgrad), bool(accumulate_wgrad))


def interleave_gate_up(gate_w: torch.Tensor, up_w: torch.Tensor) -> torch.Tensor:
    """[I, H] gate and up projection weights -> [2I, H] with rows (gate_0, up_0, gate_1, up_1, ...):
    the operand layout of linear(..., act="swiglu") (one-time, at load)."""
    return torch.stack([gate_w, up_w], dim=1).reshape(2 * gate_w.shape[0], gate_w.shape[1]).contiguous()


class _SelectRowsFn(torch.autograd.Function):
    """The rows of h [s, 1, c] that logit_mask [1, s] selects -> [M, c] (masked_select of the hidden rows,
    long_vita_megatron/core/tensor_parallel/layers.py:402-409); the gradient goes back into zeros (masked_scatter,
    :443-451).  Micro-batch 1, the reference's setting when logit_mask is used.  The row indices are computed by
    torch (host-side index op)."""

    @staticmethod
    def forward(ctx, h, logit_mask):
        s, b, c = h.shape
        if b != 1:
            raise NotImplementedError("logit-masked rows: micro-batch 1")
        idx = logit_mask.reshape(-1).nonzero().view(-1)
        ctx.save_for_backward(idx)
        ctx.s = s
        return row_gather(h.reshape(s, c), idx)

    @staticmethod
    def backward(ctx, d_sel):
        (idx,) = ctx.saved_tensors
        return row_scatter_zero(d_sel, idx, ctx.s).view(ctx.s, 1, -1), None


def select_rows(h: torch.Tensor, logit_mask: torch.Tensor) -> torch.Tensor:
    """Differentiable logit-mask row selection, h [s, 1, c] -> [M, c] (see _SelectRowsFn)."""
    return _SelectRowsFn.apply(h, logit_mask)


def masked_linear(h: torch.Tensor, weight: torch.Tensor, logit_mask: torch.Tensor, bias: Optional[torch.Tensor] = None,
                  accumulate_wgrad: bool = False):
    """Logit-masked LM head, differentiable: rows of h [s, 1, c] selected by logit_mask [1, s] -> [M, 1, vocab]
    (LinearWithGradAccumulationAndAsyncCommunication with logit_mask, layers.py:371-518, for tp = 1, no sequence
    parallelism; accumulate_wgrad is its gradient_accumulation_fusion, see linear_autograd).  Under no_grad it is the
    gather and the GEMM, nothing recorded."""
    sel = select_rows(h, logit_mask)
    return linear_autograd(sel, weight, bias, accumulate_wgrad).view(sel.shape[0], 1, weight.shape[0])


# ------------------------------------------------------------------------------------------------
# logit-masked LM head fused with the cross-entropy, chunked over the vocabulary (SURVEY.md 8f-3)
# ------------------------------------------------------------------------------------------------
def _ce_chunks(vocab: int, chunk: int):
    chunk = max(8, (chunk // 8) * 8)
    return [(v0, min(vocab, v0 + chunk)) for v0 in range(0, vocab, chunk)]


def ce_accumulate(logits: torch.Tensor, labels: torch.Tensor, run_max: torch.Tensor, run_sum: torch.Tensor, tgt: torch.Tensor,
                  col0: int) -> None:
    """Fold one vocabulary chunk of bf16 logits [M, n] (columns col0 .. col0 + n of the full row) into the running
    fp32 row statistics (in place): max, sum of exp(. - max), and the target logit where labels fall in the chunk."""
    _need_cuda_bf16(logits)
    M, n = logits.shape
    labels = _vec("ce_accumulate", "labels", labels, torch.int64, M)
    run_max, run_sum, tgt = (_vec("ce_accumulate", name, t, torch.float32, M, inplace=True)
                             for name, t in (("run_max", run_max), ("run_sum", run_sum), ("tgt", tgt)))
    _call("lv_ce_accumulate", logits.data_ptr(), logits.stride(0), labels.data_ptr(), run_max.data_ptr(), run_sum.data_ptr(),
          tgt.data_ptr(), M, n, col0)


def ce_grad(logits: torch.Tensor, labels: torch.Tensor, lse: torch.Tensor, dloss: torch.Tensor, col0: int) -> torch.Tensor:
    """In place: logits[M, n] (a vocabulary chunk) -> d_logits = (exp(logits - lse) - onehot) * dloss (bf16)."""
    _need_cuda_bf16(logits)
    M, n = logits.shape
    labels = _vec("ce_grad", "labels", labels, torch.int64, M)
    lse, dloss = _vec("ce_grad", "lse", lse, torch.float32, M), _vec("ce_grad", "dloss", dloss, torch.float32, M)
    _call("lv_ce_grad", logits.data_ptr(), logits.stride(0), logits.data_ptr(), logits.stride(0), labels.data_ptr(),
          lse.data_ptr(), dloss.data_ptr(), M, n, col0)
    return logits


def lm_head_ce_fwd(sel: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor, vocab_chunk: int = 16384):
    """Per-row cross-entropy of `sel @ weight.T` against `labels` without materialising the [M, vocab] logits:
    for every chunk of `vocab_chunk` weight rows one GEMM into a [M, chunk] bf16 buffer + `lv_ce_accumulate`.
    sel [M, c] bf16, weight [vocab, c] bf16 (vocab % 8 == 0), labels [M] int64 (negative = ignored -> loss 0).
    Returns (loss [M] fp32, lse [M] fp32).  Same arithmetic as the reference: bf16 logits (the output dtype of its
    ColumnParallelLinear), then the loss in fp32 (gpt_vl_model.py:371-414 -> logits.float())."""
    M, c = sel.shape
    V = weight.shape[0]
    dev = sel.device
    run_max = torch.full((M,), float("-inf"), dtype=torch.float32, device=dev)
    run_sum = torch.zeros((M,), dtype=torch.float32, device=dev)
    tgt = torch.zeros((M,), dtype=torch.float32, device=dev)
    if M == 0:
        return run_sum, run_sum.clone()
    labels = labels.contiguous()
    chunks = _ce_chunks(V, vocab_chunk)
    buf = torch.empty((M, chunks[0][1] - chunks[0][0]), dtype=torch.bfloat16, device=dev)
    for v0, v1 in chunks:
        lg = linear(sel, weight[v0:v1], out=buf[:, : v1 - v0])
        ce_accumulate(lg, labels, run_max, run_sum, tgt, v0)
    lse = torch.log(run_sum) + run_max
    loss = torch.where(labels >= 0, lse - tgt, torch.zeros_like(lse))
    return loss, lse


def lm_head_ce_bwd(sel: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor, lse: torch.Tensor, dloss: torch.Tensor,
                   need_dsel: bool = True, need_dw: bool = False, vocab_chunk: int = 16384,
                   main_grad: Optional[torch.Tensor] = None):
    """Backward of lm_head_ce_fwd, chunk by chunk: the chunk's logits are recomputed (one GEMM), turned into
    d_logits = (softmax - onehot) * dloss in place (`lv_ce_grad`), and contracted by the same wgmma GEMM:
    d_sel += d_logits @ W[chunk] (fp32 accumulation across chunks), dW[chunk] = d_logits^T @ sel
    (layers.py:443-456, 512-520).  Returns (d_sel [M, c] bf16 or None, dW [vocab, c] bf16 or None).  With need_dw and
    an fp32 `main_grad` [vocab, c], each chunk's dW is added to its row slice main_grad[chunk] instead
    (linear_wgrad_accumulate) and dW is None."""
    M, c = sel.shape
    V = weight.shape[0]
    dev = sel.device
    dsel = torch.zeros((M, c), dtype=torch.float32, device=dev) if need_dsel else None
    dw = torch.empty((V, c), dtype=torch.bfloat16, device=dev) if need_dw and main_grad is None else None
    if M == 0:
        if dw is not None:
            dw.zero_()
        return (None if dsel is None else dsel.to(torch.bfloat16)), dw
    labels = labels.contiguous()
    dloss = dloss.contiguous().float()
    chunks = _ce_chunks(V, vocab_chunk)
    buf = torch.empty((M, chunks[0][1] - chunks[0][0]), dtype=torch.bfloat16, device=dev)
    for v0, v1 in chunks:
        n = v1 - v0
        lg = ce_grad(linear(sel, weight[v0:v1], out=buf[:, :n]), labels, lse, dloss, v0)
        if need_dsel:
            dsel += linear(lg, weight[v0:v1].t()).float()           # the weight chunk read in place, MN-major
        if need_dw and main_grad is not None:
            linear_wgrad_accumulate(lg, sel, main_grad[v0:v1])
        elif need_dw:
            linear(lg.t(), sel.t(), out=dw[v0:v1])                  # both MN-major, the M rows are the contraction
    return (None if dsel is None else dsel.to(torch.bfloat16)), dw


class _LMHeadCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sel, weight, labels, vocab_chunk, accumulate_wgrad=False):
        labels = labels.reshape(-1)
        loss, lse = lm_head_ce_fwd(sel, weight, labels, vocab_chunk)
        ctx.save_for_backward(sel, weight, labels, lse)
        ctx.vocab_chunk, ctx.accumulate_wgrad = vocab_chunk, accumulate_wgrad
        return loss.view(1, -1)

    @staticmethod
    def backward(ctx, dloss):
        sel, weight, labels, lse = ctx.saved_tensors
        if not (ctx.accumulate_wgrad and ctx.needs_input_grad[1]):
            dsel, dw = lm_head_ce_bwd(sel, weight, labels, lse, dloss.reshape(-1), ctx.needs_input_grad[0],
                                      ctx.needs_input_grad[1], ctx.vocab_chunk)
            return dsel, dw, None, None, None
        main_grad = fused_wgrad_main_grad(weight)
        dsel, _ = lm_head_ce_bwd(sel, weight, labels, lse, dloss.reshape(-1), ctx.needs_input_grad[0], True,
                                 ctx.vocab_chunk, main_grad=main_grad)
        return dsel, fused_wgrad_dummy(weight, main_grad, sel.dtype), None, None, None


def masked_lm_head_ce(h: torch.Tensor, weight: torch.Tensor, logit_mask: torch.Tensor, labels: torch.Tensor,
                      vocab_chunk: int = 16384, accumulate_wgrad: bool = False) -> torch.Tensor:
    """GPTVLModel's training tail in one differentiable op (gpt_vl_model.py:325-339 masked_select of the hidden rows,
    :339 output_layer, :379-382 masked_select of the labels done by the caller, :412 per-token loss): h [s, 1, c],
    weight [vocab, c], logit_mask [1, s] bool, labels [1, M] (the M selected label ids) -> loss [1, M] fp32.  The
    [M, vocab] logits are never materialised (1M tokens x 152 064 would be 318 GB in bf16).  accumulate_wgrad: the
    weight gradient goes to weight.main_grad, vocabulary chunk by chunk (see linear_autograd)."""
    return _LMHeadCEFn.apply(select_rows(h, logit_mask), weight, labels, vocab_chunk, accumulate_wgrad)


# ------------------------------------------------------------------------------------------------
# differentiable building blocks of the decoder layer (training through the `--spec` layer, SURVEY.md 8f-1)
# ------------------------------------------------------------------------------------------------
def rmsnorm_bwd(x: torch.Tensor, weight: torch.Tensor, dy: torch.Tensor, eps: float = 1e-6,
                add_in: Optional[torch.Tensor] = None):
    """Gradients of rmsnorm(x, weight): returns (dx [+ add_in], dweight).  `x` is the tensor that was normalised."""
    _need_cuda_bf16(x, weight, dy, add_in)
    cols = x.shape[-1]
    x2 = _rows(x, cols)
    dy2 = _like("rmsnorm_bwd", "dy", dy, x2.shape)
    a2 = None if add_in is None else _like("rmsnorm_bwd", "add_in", add_in, x2.shape)
    weight = _param("rmsnorm_bwd", "weight", weight, cols)
    rows = x2.shape[0]
    parts = int(_lib.lib().lv_rmsnorm_bwd_partials(rows, cols))
    dw_part = torch.empty((parts, cols), dtype=torch.float32, device=x.device)
    dx = torch.empty_like(x2)
    _call("lv_rmsnorm_bwd", x2.data_ptr(), weight.data_ptr(), dy2.data_ptr(), _ptr(a2), dx.data_ptr(), dw_part.data_ptr(),
          rows, cols, float(eps))
    return dx.view(x.shape), dw_part.sum(dim=0).to(torch.bfloat16)


def swiglu_bwd(gate_up: torch.Tensor, dh: torch.Tensor):
    _need_cuda_bf16(gate_up, dh)
    inter = gate_up.shape[-1] // 2
    g2 = _rows(gate_up, 2 * inter)
    d2 = _like("swiglu_bwd", "dh", dh, (g2.shape[0], inter))
    out = torch.empty_like(g2)
    _call("lv_swiglu_bwd", g2.data_ptr(), d2.data_ptr(), out.data_ptr(), g2.shape[0], inter)
    return out.view(gate_up.shape)


class _RMSNormFn(torch.autograd.Function):
    """y = rmsnorm(x [+ residual]); with a residual also returns the sum (the new residual stream)."""

    @staticmethod
    def forward(ctx, x, residual, weight, eps):
        if residual is None:
            y, s = rmsnorm(x, weight, eps), x
        else:
            y, s = rmsnorm(x, weight, eps, residual=residual)
        ctx.save_for_backward(s, weight)
        ctx.eps, ctx.has_res = eps, residual is not None
        return (y, s) if residual is not None else y

    @staticmethod
    def backward(ctx, dy, ds=None):
        s, weight = ctx.saved_tensors
        dx, dw = rmsnorm_bwd(s, weight, dy.contiguous(), ctx.eps, add_in=ds if ctx.has_res else None)
        return dx, (dx if ctx.has_res else None), dw, None


def rmsnorm_autograd(x, weight, eps: float = 1e-6, residual=None):
    return _RMSNormFn.apply(x, residual, weight, eps)


class _SwiGLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate_up):
        ctx.save_for_backward(gate_up)
        return swiglu(gate_up)

    @staticmethod
    def backward(ctx, dh):
        (gate_up,) = ctx.saved_tensors
        return swiglu_bwd(gate_up, dh.contiguous())


def swiglu_autograd(gate_up):
    return _SwiGLUFn.apply(gate_up)


class _RopeFn(torch.autograd.Function):
    """rotate-half RoPE is linear in x: the gradient is the same rotation with -sin."""

    @staticmethod
    def forward(ctx, x, cos, sin):
        ctx.save_for_backward(cos, sin)
        return rope(x, cos, sin)

    @staticmethod
    def backward(ctx, dy):
        cos, sin = ctx.saved_tensors
        dy = dy if dy.stride(2) == 1 else dy.contiguous()
        return rope(dy, cos, -sin), None, None


def rope_autograd(x, cos, sin):
    return _RopeFn.apply(x, cos, sin)


class _LinearFn(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM; dX = dY W and dW = dY^T X reuse the same kernel, which reads the transposed
    operands (W^T, dY^T, X^T) in place as MN-major views.  With accumulate_wgrad, dW is added to weight.main_grad in
    fp32 instead (gradient-accumulation fusion, see fused_wgrad_main_grad)."""

    @staticmethod
    def forward(ctx, x, weight, bias, accumulate_wgrad=False):
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        ctx.accumulate_wgrad = accumulate_wgrad
        return linear(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        n_out, k_in = weight.shape
        dy2 = dy.reshape(-1, n_out).contiguous()
        x2 = x.reshape(-1, k_in)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = linear(dy2, weight.t()).view(x.shape)                       # [T, K] = dY [T, N] . (W^T)[K, N]^T
        if ctx.needs_input_grad[1]:
            if ctx.accumulate_wgrad:
                main_grad = fused_wgrad_main_grad(weight)
                linear_wgrad_accumulate(dy2, x2, main_grad)
                dw = fused_wgrad_dummy(weight, main_grad, dy2.dtype)
            else:
                dw = linear_wgrad(dy2, x2)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.float().sum(dim=0).to(dy2.dtype)
        return dx, dw, db, None


def linear_wgrad(dy2: torch.Tensor, x2: torch.Tensor) -> torch.Tensor:
    """dW [N, K] = dY^T [N, T] . X [T, K] on the wgmma GEMM, the token dimension T being the contraction: dY^T and X^T
    are read in place as MN-major operands, so T may be any length.  Without tokens (a context-parallel rank that
    owns no answer token) dW is zero and no GEMM runs."""
    if dy2.shape[0] == 0:
        return torch.zeros((dy2.shape[1], x2.shape[1]), dtype=dy2.dtype, device=dy2.device)
    # dY and X in place when the GEMM can read their transposes MN-major, else contiguous copies (_gemm_operand)
    (dy2, _, _), (x2, _, _) = _gemm_operand(dy2, mn_ok=False), _gemm_operand(x2, mn_ok=False)
    return linear(dy2.t(), x2.t())                                           # [N, K] = dY^T [N, T] . (X^T)[K, T]^T


def linear_wgrad_accumulate(dy2: torch.Tensor, x2: torch.Tensor, main_grad: torch.Tensor) -> torch.Tensor:
    """main_grad [N, K] fp32 += dY^T [N, T] . X [T, K], in place (`lv_gemm_wgrad_acc_f32`): the product of linear_wgrad
    with the same operands and k-order, added to main_grad in fp32 without a bf16 rounding.  main_grad may be a view
    (a row slice, or the first K columns of a wider tensor): unit column stride, a row stride that is a multiple of 4,
    16-byte aligned; elements outside it are not touched.  Without tokens nothing is launched.  Returns main_grad."""
    _need_cuda_bf16(dy2, x2)
    _need_cuda(main_grad, torch.float32)
    n_out, k_in = dy2.shape[1], x2.shape[1]
    if tuple(main_grad.shape) != (n_out, k_in):
        raise RuntimeError(f"linear_wgrad_accumulate: main_grad is {tuple(main_grad.shape)}, the weight gradient is "
                           f"[{n_out}, {k_in}]")
    if main_grad.stride(1) != 1 or main_grad.stride(0) % 4 != 0 or main_grad.data_ptr() % 16 != 0:
        raise RuntimeError(f"linear_wgrad_accumulate: main_grad (strides {main_grad.stride()}) must have unit column "
                           "stride, a row stride that is a multiple of 4 and a 16-byte aligned start")
    T = dy2.shape[0]
    if x2.shape[0] != T:
        raise ValueError(f"linear_wgrad_accumulate: dY has {T} tokens, X has {x2.shape[0]}")
    if T == 0:
        return main_grad
    (dy2, _, lda), (x2, _, ldw) = _gemm_operand(dy2, mn_ok=False), _gemm_operand(x2, mn_ok=False)
    ev0 = _TIMER.start() if _TIMER is not None else None
    _call("lv_gemm_wgrad_acc_f32", dy2.data_ptr(), x2.data_ptr(), main_grad.data_ptr(), n_out, k_in, T, lda, ldw,
          main_grad.stride(0), 1, 1)
    if ev0 is not None:
        _TIMER.stop("gemm_bf16", 2.0 * n_out * k_in * T, ev0)
    return main_grad


def fused_wgrad_main_grad(weight: torch.Tensor) -> torch.Tensor:
    """The fp32 `main_grad` a weight gradient is accumulated into under Megatron's gradient_accumulation_fusion
    (long_vita_megatron/core/tensor_parallel/layers.py:486-497; Megatron's DDP wrapper allocates it)."""
    main_grad = getattr(weight, "main_grad", None)
    if main_grad is None:
        raise RuntimeError(f"gradient_accumulation_fusion: the trainable weight of shape {tuple(weight.shape)} has no "
                           "`main_grad` to accumulate into (it is allocated by Megatron's DistributedDataParallel)")
    if main_grad.dtype != torch.float32:
        raise NotImplementedError(f"gradient_accumulation_fusion: main_grad is {main_grad.dtype}; only an fp32 "
                                  "main_grad is supported (Megatron's with --bf16)")
    return main_grad


def fused_wgrad_dummy(weight: torch.Tensor, main_grad: torch.Tensor, dtype: torch.dtype) -> Optional[torch.Tensor]:
    """The gradient returned for a weight whose gradient went to main_grad (layers.py:499-518): None when the weight has
    no `grad_added_to_main_grad` attribute; otherwise a main_grad-shaped tensor - zeros with `zero_out_wgrad`, else
    uninitialised - and grad_added_to_main_grad is set."""
    if not hasattr(weight, "grad_added_to_main_grad"):
        return None
    make = torch.zeros if getattr(weight, "zero_out_wgrad", False) else torch.empty
    weight.grad_added_to_main_grad = True
    return make(main_grad.shape, dtype=dtype, device=main_grad.device)


def linear_autograd(x, weight, bias=None, accumulate_wgrad: bool = False):
    """Differentiable linear (see _LinearFn).  accumulate_wgrad: the weight gradient is added to weight.main_grad
    (fp32) and the returned gradient follows fused_wgrad_dummy; the bias gradient is unchanged."""
    if accumulate_wgrad:        # otherwise the node keeps three inputs, as a backward written for x, weight, bias expects
        return _LinearFn.apply(x, weight, bias, True)
    return _LinearFn.apply(x, weight, bias)


def patch_embed(images: torch.Tensor, w_pad: torch.Tensor, bias: Optional[torch.Tensor], cls: torch.Tensor,
                pos: torch.Tensor, patch: int):
    """images [n,3,S,S] -> [n, 1 + (S/patch)^2, C] (conv-as-GEMM + cls + position embedding).
    `w_pad` is the conv weight flattened to [C, 3*patch*patch] and zero-padded to a multiple of 64."""
    _need_cuda_bf16(images, w_pad, bias, cls, pos)
    images = images.contiguous()
    n, _, size, _ = images.shape
    Cc = w_pad.shape[0]
    P = (size // patch) ** 2
    S = P + (0 if cls is None else 1)
    w_pad = _like("patch_embed", "w_pad", w_pad, (Cc, (3 * patch * patch + 63) // 64 * 64))
    bias, cls = _param("patch_embed", "bias", bias, Cc), _param("patch_embed", "cls", cls, Cc)
    pos = _param("patch_embed", "pos", pos, S * Cc)
    ws_bytes = int(_lib.lib().lv_patch_embed_ws_bytes(n, size, patch, Cc))
    ws = torch.empty(ws_bytes // 2, dtype=torch.bfloat16, device=images.device)
    out = torch.empty((n, S, Cc), dtype=torch.bfloat16, device=images.device)
    _call("lv_patch_embed", images.data_ptr(), w_pad.data_ptr(), _ptr(bias), _ptr(cls), pos.data_ptr(), out.data_ptr(),
          ws.data_ptr(), n, size, patch, Cc)
    return out


def pad_patch_weight(conv_weight: torch.Tensor) -> torch.Tensor:
    """[C, 3, ps, ps] conv weight -> [C, Kpad] GEMM operand (one-time, at load)."""
    Cc = conv_weight.shape[0]
    flat = conv_weight.reshape(Cc, -1)
    k = flat.shape[1]
    kpad = (k + 63) // 64 * 64
    out = torch.zeros((Cc, kpad), dtype=conv_weight.dtype, device=conv_weight.device)
    out[:, :k] = flat
    return out


# ------------------------------------------------------------------------------------------------
# differentiable building blocks of the vision tower and the projector (training InternViT through
# MegatronVisionModel, pretrain_long_vita.py:310-596).  Each backward is a kernel of liblvb200.so; the per-column
# gradients (LayerNorm weight / bias, layer scale) come back as fp32 partial rows that are added here, and the
# bias-like sums (conv bias, class token, position embedding, linear bias) are fp32 sums over tokens, as in
# _LinearFn.
# ------------------------------------------------------------------------------------------------
def layernorm_bwd(x: torch.Tensor, weight: torch.Tensor, dy: torch.Tensor, eps: float = 1e-6,
                  add_in: Optional[torch.Tensor] = None, need_dx: bool = True):
    """Gradients of layernorm(x, weight, bias): returns (dx [+ add_in], dweight, dbias); dx is None (and not computed)
    with need_dx=False."""
    if not need_dx and add_in is not None:
        raise ValueError("layernorm_bwd: add_in needs dx")
    _need_cuda_bf16(x, weight, dy, add_in)
    cols = x.shape[-1]
    x2 = _rows(x, cols)
    dy2 = _like("layernorm_bwd", "dy", dy, x2.shape)
    a2 = None if add_in is None else _like("layernorm_bwd", "add_in", add_in, x2.shape)
    weight = _param("layernorm_bwd", "weight", weight, cols)
    rows = x2.shape[0]
    parts = int(_lib.lib().lv_layernorm_bwd_partials(rows, cols))
    dw_part = torch.empty((parts, cols), dtype=torch.float32, device=x.device)
    db_part = torch.empty((parts, cols), dtype=torch.float32, device=x.device)
    dx = torch.empty_like(x2) if need_dx else None
    _call("lv_layernorm_bwd", x2.data_ptr(), weight.data_ptr(), dy2.data_ptr(), _ptr(a2), _ptr(dx), dw_part.data_ptr(),
          db_part.data_ptr(), rows, cols, float(eps))
    return (None if dx is None else dx.view(x.shape)), dw_part.sum(dim=0).to(torch.bfloat16), db_part.sum(dim=0).to(torch.bfloat16)


def gelu_bwd(pre: torch.Tensor, dy: torch.Tensor, approximate: str = "none"):
    """dx = dy * gelu'(pre); `approximate` as in bias_gelu ("none" = erf, "tanh")."""
    _need_cuda_bf16(pre, dy)
    cols = pre.shape[-1]
    p2 = _rows(pre, cols)
    d2 = _like("gelu_bwd", "dy", dy, p2.shape)
    dx = torch.empty_like(p2)
    _call("lv_gelu_bwd", p2.data_ptr(), d2.data_ptr(), dx.data_ptr(), p2.shape[0], cols, 1 if approximate == "tanh" else 0)
    return dx.view(pre.shape)


def ls_residual_bwd(dout: torch.Tensor, y: torch.Tensor, ls: torch.Tensor):
    """Gradients of ls_residual(x, y, ls) (no bias) with respect to y and ls: (bf16(dout * ls), sum_rows dout * y).
    The gradient of x is dout itself."""
    _need_cuda_bf16(dout, y, ls)
    cols = y.shape[-1]
    y2 = _rows(y, cols)
    d2 = _like("ls_residual_bwd", "dout", dout, y2.shape)
    ls = _param("ls_residual_bwd", "ls", ls, cols)
    rows = y2.shape[0]
    parts = int(_lib.lib().lv_ls_residual_bwd_partials(rows, cols))
    dls_part = torch.empty((parts, cols), dtype=torch.float32, device=y.device)
    dy = torch.empty_like(y2)
    _call("lv_ls_residual_bwd", d2.data_ptr(), y2.data_ptr(), ls.data_ptr(), dy.data_ptr(), dls_part.data_ptr(), rows, cols)
    return dy.view(y.shape), dls_part.sum(dim=0).to(torch.bfloat16)


def pixel_shuffle_bwd(dout: torch.Tensor, hw: int, has_cls: bool):
    """[n, (hw/2)^2, 4c] -> [n, (1 +) hw*hw, c]: the inverse permutation of pixel_shuffle (class-token rows zero)."""
    _need_cuda_bf16(dout)
    if dout.dim() != 3 or dout.shape[1] != (hw // 2) ** 2:
        raise ValueError(f"pixel_shuffle_bwd: dout {tuple(dout.shape)} is not [n, ({hw}/2)^2, 4c]")
    dout = dout.contiguous()
    n, _, c4 = dout.shape
    c = c4 // 4
    dx = torch.empty((n, hw * hw + (1 if has_cls else 0), c), dtype=torch.bfloat16, device=dout.device)
    _call("lv_pixel_shuffle_bwd", dout.data_ptr(), dx.data_ptr(), n, hw, c, 1 if has_cls else 0)
    return dx


def patch_im2col(images: torch.Tensor, patch: int, kpad: int):
    """images [n, 3, S, S] -> col [n * (S/patch)^2, kpad]: each patch's pixels in (channel, y, x) order, zero-padded."""
    _need_cuda_bf16(images)
    images = images.contiguous()
    n, _, size, _ = images.shape
    col = torch.empty((n * (size // patch) ** 2, kpad), dtype=torch.bfloat16, device=images.device)
    _call("lv_patch_im2col", images.data_ptr(), col.data_ptr(), n, size, patch, kpad)
    return col


class _LayerNormFn(torch.autograd.Function):
    """y = layernorm(x).  With `passthrough`, also returns x itself as the residual stream: the gradient arriving on
    that second output is added to dx inside the backward kernel (`add_in`), so the residual branch of a pre-norm
    block costs no separate add."""

    @staticmethod
    def forward(ctx, x, weight, bias, eps, passthrough):
        ctx.save_for_backward(x, weight)
        ctx.eps, ctx.passthrough = eps, passthrough
        y = layernorm(x, weight, bias, eps)
        return (y, x.view_as(x)) if passthrough else y

    @staticmethod
    def backward(ctx, dy, ds=None):
        x, weight = ctx.saved_tensors
        need_dx = ctx.needs_input_grad[0]
        dx, dw, db = layernorm_bwd(x, weight, dy.contiguous(), ctx.eps, add_in=ds if ctx.passthrough and need_dx else None,
                                   need_dx=need_dx)
        return dx, dw, db, None, None


def layernorm_autograd(x, weight, bias, eps: float = 1e-6, passthrough: bool = False):
    """Differentiable LayerNorm over the last dim; `passthrough=True` returns (y, x) (see _LayerNormFn)."""
    return _LayerNormFn.apply(x, weight, bias, eps, passthrough)


class _GeluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pre, approximate):
        ctx.save_for_backward(pre)
        ctx.approximate = approximate
        return bias_gelu(pre, None, approximate)

    @staticmethod
    def backward(ctx, dy):
        (pre,) = ctx.saved_tensors
        return gelu_bwd(pre, dy.contiguous(), ctx.approximate), None


def gelu_autograd(pre, approximate: str = "none"):
    """gelu(pre) keeping the bf16 pre-activation for the backward (fc1 runs with act = 0 before it in training)."""
    return _GeluFn.apply(pre, approximate)


class _LSResidualFn(torch.autograd.Function):
    """out = x + y * ls (bias-free; the ViT adds its biases in the GEMM epilogue)."""

    @staticmethod
    def forward(ctx, x, y, ls):
        ctx.save_for_backward(y, ls)
        return ls_residual(x, y, ls)

    @staticmethod
    def backward(ctx, dout):
        y, ls = ctx.saved_tensors
        dout = dout.contiguous()
        dy = dls = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dy, dls = ls_residual_bwd(dout, y, ls)
        return dout, dy, dls


def ls_residual_autograd(x, y, ls):
    return _LSResidualFn.apply(x, y, ls)


class _PixelShuffleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, hw, has_cls):
        ctx.hw, ctx.has_cls = hw, has_cls
        return pixel_shuffle(x, hw, has_cls)

    @staticmethod
    def backward(ctx, dout):
        return pixel_shuffle_bwd(dout, ctx.hw, ctx.has_cls), None, None


def pixel_shuffle_autograd(x, hw: int, has_cls: bool):
    """Differentiable drop-cls + pixel-shuffle x0.5 ([n, (1 +) hw*hw, c] -> [n, (hw/2)^2, 4c])."""
    return _PixelShuffleFn.apply(x, hw, has_cls)


class _PatchEmbedFn(torch.autograd.Function):
    """out = cat(cls, conv(images)) + pos.  Saves only the images (the im2col matrix is rebuilt in the backward);
    the conv weight gradient is dW[C, Kpad] = dP^T . col on the wgmma GEMM, with the padding columns dropped."""

    @staticmethod
    def forward(ctx, images, conv_w, conv_b, cls, pos, patch, accumulate_wgrad=False):
        w_pad = pad_patch_weight(conv_w)
        ctx.save_for_backward(images, conv_w if accumulate_wgrad else None)
        ctx.patch, ctx.kpad, ctx.w_shape = patch, w_pad.shape[1], conv_w.shape
        ctx.cls_shape, ctx.pos_shape = cls.shape, pos.shape
        ctx.accumulate_wgrad = accumulate_wgrad
        return patch_embed(images, w_pad, conv_b, cls.reshape(-1), pos, patch)

    @staticmethod
    def backward(ctx, dout):
        images, conv_w = ctx.saved_tensors
        n, s, c = dout.shape
        d = dout.contiguous()
        dw = db = dcls = dpos = None
        dp = d[:, 1:].reshape(n * (s - 1), c)
        if ctx.needs_input_grad[1]:
            col = patch_im2col(images, ctx.patch, ctx.kpad)
            k = ctx.w_shape[1] * ctx.w_shape[2] * ctx.w_shape[3]
            if ctx.accumulate_wgrad:
                # only the k real im2col columns: the padding columns of the [C, kpad] product never reach main_grad
                main_grad = fused_wgrad_main_grad(conv_w)
                linear_wgrad_accumulate(dp, col[:, :k], main_grad.view(ctx.w_shape[0], k))
                dw = fused_wgrad_dummy(conv_w, main_grad, d.dtype)
            else:
                dw = linear_wgrad(dp, col)[:, :k].reshape(ctx.w_shape)
        if ctx.needs_input_grad[2]:
            db = dp.float().sum(dim=0).to(d.dtype)
        if ctx.needs_input_grad[3]:
            dcls = d[:, 0].float().sum(dim=0).to(d.dtype).reshape(ctx.cls_shape)
        if ctx.needs_input_grad[4]:
            dpos = d.float().sum(dim=0).to(d.dtype).reshape(ctx.pos_shape)
        return None, dw, db, dcls, dpos, None, None


def patch_embed_autograd(images, conv_w, conv_b, cls, pos, patch: int, accumulate_wgrad: bool = False):
    """Differentiable InternViT embedding: images [n, 3, S, S], conv_w [C, 3, patch, patch], conv_b [C], cls (C
    elements, e.g. [1, 1, C]), pos [1 + (S/patch)^2, C] -> [n, 1 + (S/patch)^2, C].  Gradients: conv weight, conv bias,
    class token (sum over frames of row 0), position embedding (sum over frames); none for the images.
    accumulate_wgrad: the conv weight gradient goes to conv_w.main_grad (see linear_autograd)."""
    return _PatchEmbedFn.apply(images, conv_w, conv_b, cls, pos, patch, accumulate_wgrad)


class _ViTAttentionFn(torch.autograd.Function):
    """Non-causal attention over the output of the fused QKV GEMM, qkv [n, S, 3C] with Megatron's per-head row
    interleave [H, (q, k, v), D]: q / k / v are strided views of it in both directions, and the backward writes dQ / dK
    / dV through the same strides into one dQKV buffer that is the gradient of qkv (no re-layout, no stacking)."""

    @staticmethod
    def forward(ctx, qkv, heads, scale):
        n, s, c3 = qkv.shape
        d = c3 // (3 * heads)
        v5 = qkv.view(n, s, heads, 3, d)
        out, lse = attention_fwd(v5[:, :, :, 0], v5[:, :, :, 1], v5[:, :, :, 2], causal=False, scale=scale, return_lse=True)
        ctx.save_for_backward(qkv, out, lse)
        ctx.heads, ctx.scale = heads, scale
        return out.view(n, s, heads * d)

    @staticmethod
    def backward(ctx, d_out):
        qkv, out, lse = ctx.saved_tensors
        n, s, c3 = qkv.shape
        h = ctx.heads
        d = c3 // (3 * h)
        v5 = qkv.view(n, s, h, 3, d)
        dqkv = torch.empty_like(qkv)
        g5 = dqkv.view(n, s, h, 3, d)
        attention_bwd(d_out.reshape(n, s, h, d).contiguous(), v5[:, :, :, 0], v5[:, :, :, 1], v5[:, :, :, 2], out, lse,
                      causal=False, scale=ctx.scale, dq=g5[:, :, :, 0], dk=g5[:, :, :, 1], dv=g5[:, :, :, 2])
        return dqkv, None, None


def vit_attention(qkv, heads: int, scale: Optional[float] = None):
    """Differentiable ViT self-attention on qkv [n, S, 3C] ([H, 3, D] columns) -> [n, S, C] (see _ViTAttentionFn)."""
    return _ViTAttentionFn.apply(qkv, heads, scale)
