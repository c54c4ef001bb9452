"""Host-logic harness for CPU tests - TEST INFRASTRUCTURE ONLY, never imported by the product package.

The Python layers above the C ABI (weight re-layouts, index translation, argument handling, the
order in which operators are composed) are host logic: it can be wrong while every kernel is right.
To check it on a box without a GPU, `oracle_ops()` temporarily replaces the operator wrappers of
`long_vita_b200.ops` (each of which normally calls liblvb200.so and refuses non-CUDA tensors) by the
CPU oracle restatements with the same signatures.  What such a test proves is the composition - it
says nothing about the kernels, whose parity tests are the `-m gpu` files and run the real library.
Outside this context manager the product path is untouched and still fails loudly without CUDA.
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from oracle import ops as O


def _bf(x):
    return x.to(torch.bfloat16)


def _attention_fwd(q, k, v, *, causal, scale=None, layout="bshd", return_lse=False, q_seg_len=None, q_seg_pos=None,
                   kv_pos0=0, out=None):
    perm = {"bshd": (0, 1, 2, 3), "sbhd": (1, 0, 2, 3), "bhsd": (0, 2, 1, 3)}[layout]
    qv, kv, vv = (t.permute(perm) for t in (q, k, v))
    sq, sk = qv.shape[1], kv.shape[1]
    q_pos = None
    if q_seg_len is not None and q_seg_pos is not None:
        q_pos = torch.cat([torch.arange(q_seg_len) + q_seg_pos[i] for i in range(sq // q_seg_len)])
    elif q_seg_pos is not None:
        q_pos = torch.arange(sq) + q_seg_pos[0]
    o, lse = O.attention(qv, kv, vv, causal=causal, scale=scale, q_pos=q_pos, kv_pos=torch.arange(sk) + kv_pos0)
    inv = [perm.index(i) for i in range(4)]
    o = _bf(o).permute(inv)
    if out is not None:
        out.copy_(o)
        o = out
    return (o, lse) if return_lse else o


def _seg_pos(sq, q_seg_len, q_seg_pos):
    if q_seg_len is not None and q_seg_pos is not None:
        return torch.cat([torch.arange(q_seg_len) + q_seg_pos[i] for i in range(sq // q_seg_len)])
    if q_seg_pos is not None:
        return torch.arange(sq) + q_seg_pos[0]
    return None


def _attention_bwd(d_out, q, k, v, out, lse, *, causal, scale=None, q_seg_len=None, q_seg_pos=None, kv_pos0=0):
    with torch.enable_grad():      # the oracle differentiates by autograd; this runs inside an autograd backward
        dq, dk, dv = O.attention_grads(q, k, v, d_out, causal=causal, scale=scale,
                                       q_pos=_seg_pos(q.shape[1], q_seg_len, q_seg_pos), kv_pos=torch.arange(k.shape[1]) + kv_pos0)
    return _bf(dq), _bf(dk), _bf(dv)


def _decode_merge(o_part, lse_part, return_lse=False):
    n, G, hkv, d = o_part.shape
    lse = torch.logsumexp(lse_part, dim=0)                                            # [hkv, G]
    w = torch.exp(lse_part - lse.unsqueeze(0)).permute(0, 2, 1).unsqueeze(-1)          # [n, G, hkv, 1]
    out = _bf((o_part.float() * w).sum(dim=0)).transpose(0, 1).reshape(hkv * G, d)
    return (out, lse.reshape(hkv * G)) if return_lse else out


def _rmsnorm_bwd(x, weight, dy, eps=1e-6, add_in=None):
    with torch.enable_grad():
        xf = x.detach().float().requires_grad_(True)
        wf = weight.detach().float().requires_grad_(True)
        y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * wf
        y.backward(dy.float())
    dx = xf.grad if add_in is None else xf.grad + add_in.float()
    return _bf(dx), _bf(wf.grad)


def _swiglu_bwd(gate_up, dh):
    with torch.enable_grad():
        gu = gate_up.detach().float().requires_grad_(True)
        O.swiglu(gu).backward(dh.float())
    return _bf(gu.grad)


def _rmsnorm(x, weight, eps=1e-6, residual=None):
    if residual is None:
        return O.rmsnorm(x, weight, eps)
    s = _bf(x.float() + residual.float())
    return O.rmsnorm(s, weight, eps), s


def _rope_table(pos, inv_freq):
    return O.rope_tables(pos.view(-1), inv_freq, torch.bfloat16)


def _rope(x, cos, sin, out=None):
    y = _bf(x.float() * cos.float()[:, None, :] +
            torch.cat((-x.float()[..., x.shape[-1] // 2:], x.float()[..., : x.shape[-1] // 2]), -1) * sin.float()[:, None, :])
    if out is None:
        return y
    out.copy_(y)
    return out


def _linear(x, weight, bias=None, act=None, out=None):
    y = x.float().reshape(-1, x.shape[-1]) @ weight.float().t()
    if bias is not None:
        y = y + bias.float()
    if act == "gelu":
        y = F.gelu(y)
    elif act == "gelu_tanh":
        y = F.gelu(y, approximate="tanh")
    elif act == "swiglu":                      # rows interleaved (gate_i, up_i)
        y = F.silu(_bf(y[:, 0::2]).float()) * _bf(y[:, 1::2]).float()
    y = _bf(y)
    if out is not None:
        out.view(y.shape).copy_(y)
        y = out
    return y.view(*x.shape[:-1], y.shape[-1])


def _pixel_shuffle(x, hw, has_cls):
    n, _, c = x.shape
    t = x[:, 1:] if has_cls else x
    return O.pixel_shuffle_half(t.reshape(n, hw, hw, c)).reshape(n, (hw // 2) ** 2, 4 * c)


def _patch_embed(images, w_pad, bias, cls, pos, patch):
    C = w_pad.shape[0]
    w = w_pad[:, : 3 * patch * patch].reshape(C, 3, patch, patch)
    pe = F.conv2d(images.float(), w.float(), None if bias is None else bias.float(), stride=patch).flatten(2).transpose(1, 2)
    if cls is not None:
        pe = torch.cat([cls.float().reshape(1, 1, -1).expand(pe.shape[0], 1, -1), pe], dim=1)
    return _bf(pe + pos.float().reshape(1, -1, C)).contiguous()      # the kernel writes a fresh contiguous [n, S, C]


def _row_scatter_zero(x, idx, n_rows_out):
    out = torch.zeros((n_rows_out, x.shape[1]), dtype=x.dtype)
    out[idx.view(-1)] = x
    return out


def _ce_accumulate(logits, labels, run_max, run_sum, tgt, col0):
    x = logits.float()
    m_new = torch.maximum(run_max, x.max(dim=1).values)
    run_sum.copy_(torch.where(torch.isinf(run_max), torch.zeros_like(run_sum), run_sum * torch.exp(run_max - m_new))
                  + torch.exp(x - m_new[:, None]).sum(dim=1))
    run_max.copy_(m_new)
    lab = labels - col0
    hit = (lab >= 0) & (lab < x.shape[1])
    tgt[hit] = x[hit.nonzero().view(-1), lab[hit]]


def _ce_grad(logits, labels, lse, dloss, col0):
    x = logits.float()
    p = torch.exp(x - lse[:, None])
    lab = labels - col0
    hit = (lab >= 0) & (lab < x.shape[1])
    p[hit.nonzero().view(-1), lab[hit]] -= 1.0
    g = torch.where(labels < 0, torch.zeros_like(dloss), dloss)
    logits.copy_(_bf(p * g[:, None]))
    return logits


SUBSTITUTES = {
    "ce_accumulate": _ce_accumulate,
    "ce_grad": _ce_grad,
    "attention_fwd": _attention_fwd,
    "attention_bwd": _attention_bwd,
    "decode_merge": _decode_merge,
    "rmsnorm": _rmsnorm,
    "rmsnorm_bwd": _rmsnorm_bwd,
    "swiglu_bwd": _swiglu_bwd,
    "layernorm": lambda x, w, b, eps=1e-6: O.layernorm(x, w, b, eps),
    "rope_table": _rope_table,
    "rope": _rope,
    "swiglu": lambda gu: _bf(O.swiglu(gu.float())),
    "bias_gelu": lambda x, bias=None, approximate="none": _bf(O.bias_gelu(x.float(), None if bias is None else bias.float(), approximate)),
    "ls_residual": lambda x, y, ls=None, bias=None: _bf(O.ls_residual(x.float(), y.float(), None if ls is None else ls.float(),
                                                                         None if bias is None else bias.float())),
    "pixel_shuffle": _pixel_shuffle,
    "embed_scatter": lambda ids, table, feat=None, dst_idx=None, src_idx=None: O.embed_scatter(ids, table, feat, dst_idx, src_idx),
    "row_gather": lambda x, idx: x[idx.view(-1)].clone(),
    "row_scatter_zero": _row_scatter_zero,
    "linear": _linear,
    "patch_embed": _patch_embed,
    # composite wrappers (masked_linear, masked_lm_head_ce) keep their own host logic and only lose
    # the "must be a CUDA tensor" guard
    "_need_cuda_bf16": lambda *ts: None,
    "_need_cuda": lambda t, dtype: None,
}


@contextlib.contextmanager
def oracle_ops():
    """Within the block, long_vita_b200.ops.<op> are the CPU oracle restatements (see module doc)."""
    from long_vita_b200 import ops

    saved = {name: getattr(ops, name) for name in SUBSTITUTES}
    try:
        for name, fn in SUBSTITUTES.items():
            setattr(ops, name, fn)
        yield ops
    finally:
        for name, fn in saved.items():
            setattr(ops, name, fn)
