"""CPU oracle of document-masked attention over one packed row - TEST INFRASTRUCTURE ONLY.

Packed training samples (`--reset-position-ids --reset-attention-mask`) attend only inside their own sample: key j is
visible to query i iff both lie in the same document of cu_seqlens = [0, c_1, ..., c_n = S] and j <= i.  This is the
mask of Megatron's get_ltor_masks_and_position_ids(reset_attention_mask=True) (long_vita_megatron/training/utils.py
:192-249, pinned against the reference's own output in tests/test_packed_docs_host.py) and of
flash_attn_varlen_func(causal=True) over the documents.  Arithmetic as in `oracle.ops.attention` (fp32 scores and
softmax, GQA without expansion, scale 1/sqrt(d)) with that mask made explicit.

`packed_oracle_ops()` is `tests.hostlogic.oracle_ops()` whose attention substitutes also accept `cu_seqlens`, so the
composed modules run on the CPU with packed rows.
"""
from __future__ import annotations

import contextlib
import math
from typing import Optional

import torch

from tests import hostlogic


def document_mask(cu_seqlens, seq_len: int) -> torch.Tensor:
    """[S, S] bool, True = hidden (Megatron returns `mask < 0.5`, the same convention)."""
    cu = torch.as_tensor(cu_seqlens, dtype=torch.int64).reshape(-1).cpu()
    pos = torch.arange(seq_len, dtype=torch.int64)
    doc = torch.bucketize(pos, cu[1:], right=True)           # document of each position
    return (doc[None, :] != doc[:, None]) | (pos[None, :] > pos[:, None])


def attention(q, k, v, cu_seqlens, *, scale: Optional[float] = None, head_chunk: int = 8):
    """q [1, S, hq, d], k / v [1, S, hkv, d] -> (out [1, S, hq, d] fp32, lse [1, hq, S] fp32)."""
    b, sq, hq, d = q.shape
    assert b == 1 and k.shape[1] == sq
    hidden = document_mask(cu_seqlens, sq)
    g = hq // k.shape[2]
    scale = 1.0 / math.sqrt(d) if scale is None else scale
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    out = torch.empty((b, hq, sq, d), dtype=torch.float32)
    lse = torch.empty((b, hq, sq), dtype=torch.float32)
    for h0 in range(0, hq, head_chunk):
        h1 = min(hq, h0 + head_chunk)
        kvh = torch.arange(h0, h1) // g
        s = (torch.matmul(qf[:, h0:h1], kf[:, kvh].transpose(-1, -2)) * scale).masked_fill(hidden, float("-inf"))
        l = torch.logsumexp(s, dim=-1)
        out[:, h0:h1] = torch.matmul(torch.nan_to_num(torch.exp(s - l.unsqueeze(-1)), nan=0.0), vf[:, kvh])
        lse[:, h0:h1] = l
    return out.permute(0, 2, 1, 3).contiguous(), lse


def attention_grads(q, k, v, d_out, cu_seqlens, *, scale: Optional[float] = None):
    """dq, dk, dv of `attention` by fp32 autograd over the same definition."""
    qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    b, sq, hq, d = qf.shape
    g = hq // kf.shape[2]
    scale = 1.0 / math.sqrt(d) if scale is None else scale
    with torch.enable_grad():
        s = torch.einsum("bqhd,bkhd->bhqk", qf, kf.repeat_interleave(g, dim=2)) * scale
        s = s.masked_fill(document_mask(cu_seqlens, sq), float("-inf"))
        p = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
        torch.einsum("bhqk,bkhd->bqhd", p, vf.repeat_interleave(g, dim=2)).backward(d_out.float())
    return qf.grad, kf.grad, vf.grad


_PERM = {"bshd": (0, 1, 2, 3), "sbhd": (1, 0, 2, 3), "bhsd": (0, 2, 1, 3)}


def _attention_fwd(q, k, v, *, causal, scale=None, layout="bshd", return_lse=False, out=None, cu_seqlens=None, **kw):
    if cu_seqlens is None:
        return hostlogic.SUBSTITUTES["attention_fwd"](q, k, v, causal=causal, scale=scale, layout=layout,
                                                      return_lse=return_lse, out=out, **kw)
    if not causal:
        raise NotImplementedError("packed documents without a causal mask are not supported")
    perm = _PERM[layout]
    o, lse = attention(*(t.permute(perm) for t in (q, k, v)), cu_seqlens, scale=scale)
    o = o.to(torch.bfloat16).permute([perm.index(i) for i in range(4)])
    if out is not None:
        out.copy_(o)
        o = out
    return (o, lse) if return_lse else o


def _attention_bwd(d_out, q, k, v, out, lse, *, causal, scale=None, cu_seqlens=None, **kw):
    if cu_seqlens is None:
        return hostlogic.SUBSTITUTES["attention_bwd"](d_out, q, k, v, out, lse, causal=causal, scale=scale, **kw)
    dq, dk, dv = attention_grads(q, k, v, d_out, cu_seqlens, scale=scale)
    return dq.to(torch.bfloat16), dk.to(torch.bfloat16), dv.to(torch.bfloat16)


@contextlib.contextmanager
def packed_oracle_ops():
    """hostlogic.oracle_ops() with attention substitutes that also take `cu_seqlens` (see module doc)."""
    with hostlogic.oracle_ops() as ops:
        ops.attention_fwd, ops.attention_bwd = _attention_fwd, _attention_bwd    # restored by oracle_ops on exit
        yield ops
