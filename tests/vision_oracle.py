"""CPU oracle forms of the vision-tower training operators - TEST INFRASTRUCTURE ONLY.

`vision_oracle_ops()` is `tests.hostlogic.oracle_ops()` plus CPU restatements of the operators the trainable vision
side (`long_vita_b200.megatron.vision_model.B200VisionModel`) calls: the forward wrappers it shares with inference
(linear, layernorm, bias_gelu, ls_residual, pixel_shuffle, patch_embed, attention) and the new backward wrappers
(layernorm_bwd, gelu_bwd, ls_residual_bwd, pixel_shuffle_bwd, patch_im2col, attention_bwd into caller buffers).
Unlike the hostlogic forms, these compute in fp32 and return the dtype of their input, so a model with fp32
parameters runs the whole composition in fp32 and can be held to the fp32 reference fixture; with bf16 inputs they
round to bf16 like the kernels.  `calls` counts how often each backward operator ran inside the block.
"""
from __future__ import annotations

import contextlib
from collections import Counter

import torch
import torch.nn.functional as F

from oracle import ops as O
from tests import hostlogic

calls: Counter = Counter()

BACKWARD_OPS = ("layernorm_bwd", "gelu_bwd", "ls_residual_bwd", "pixel_shuffle_bwd", "patch_im2col", "attention_bwd")


def _linear(x, weight, bias=None, act=None, out=None):
    y = x.float().reshape(-1, x.shape[-1]) @ weight.float().t()
    if bias is not None:
        y = y + bias.float()
    if act == "gelu":
        y = F.gelu(y)
    elif act is not None:
        raise NotImplementedError(act)
    y = y.to(x.dtype)
    if out is not None:
        out.view(y.shape).copy_(y)
        y = out
    return y.view(*x.shape[:-1], y.shape[-1])


def _layernorm(x, w, b, eps=1e-6):
    return F.layer_norm(x.float(), (x.shape[-1],), w.float(), None if b is None else b.float(), eps).to(x.dtype)


def _layernorm_bwd(x, weight, dy, eps=1e-6, add_in=None, need_dx=True):
    calls["layernorm_bwd"] += 1
    if not need_dx:
        calls["layernorm_bwd_no_dx"] += 1
    with torch.enable_grad():
        xf = x.detach().float().requires_grad_(True)
        wf = weight.detach().float().requires_grad_(True)
        bf = torch.zeros_like(wf, requires_grad=True)
        F.layer_norm(xf, (x.shape[-1],), wf, bf, eps).backward(dy.float())
    dx = xf.grad if add_in is None else xf.grad + add_in.float()
    return (dx.to(x.dtype) if need_dx else None), wf.grad.to(weight.dtype), bf.grad.to(weight.dtype)


def _bias_gelu(x, bias=None, approximate="none"):
    return O.bias_gelu(x.float(), None if bias is None else bias.float(), approximate).to(x.dtype)


def _gelu_bwd(pre, dy, approximate="none"):
    calls["gelu_bwd"] += 1
    with torch.enable_grad():
        p = pre.detach().float().requires_grad_(True)
        F.gelu(p, approximate=approximate).backward(dy.float())
    return p.grad.to(pre.dtype)


def _ls_residual(x, y, ls=None, bias=None):
    return O.ls_residual(x.float(), y.float(), None if ls is None else ls.float(), None if bias is None else bias.float()).to(x.dtype)


def _ls_residual_bwd(dout, y, ls):
    calls["ls_residual_bwd"] += 1
    d = dout.float().reshape(-1, y.shape[-1])
    return (d * ls.float()).to(y.dtype).view(y.shape), (d * y.float().reshape(d.shape)).sum(dim=0).to(ls.dtype)


def _pixel_shuffle_bwd(dout, hw, has_cls):
    calls["pixel_shuffle_bwd"] += 1
    n, _, c4 = dout.shape
    c = c4 // 4
    g = dout.reshape(n, hw // 2, hw // 2, 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, hw * hw, c)   # inverse of O.pixel_shuffle_half
    if has_cls:
        g = torch.cat([torch.zeros((n, 1, c), dtype=dout.dtype), g], dim=1)
    return g.contiguous()


def _patch_embed(images, w_pad, bias, cls, pos, patch):
    C = w_pad.shape[0]
    w = w_pad[:, : 3 * patch * patch].reshape(C, 3, patch, patch)
    pe = F.conv2d(images.float(), w.float(), None if bias is None else bias.float(), stride=patch).flatten(2).transpose(1, 2)
    if cls is not None:
        pe = torch.cat([cls.float().reshape(1, 1, -1).expand(pe.shape[0], 1, -1), pe], dim=1)
    return (pe + pos.float().reshape(1, -1, C)).to(images.dtype).contiguous()


def _patch_im2col(images, patch, kpad):
    calls["patch_im2col"] += 1
    n, c, s, _ = images.shape
    g = s // patch
    col = images.reshape(n, c, g, patch, g, patch).permute(0, 2, 4, 1, 3, 5).reshape(n * g * g, c * patch * patch)
    return F.pad(col, (0, kpad - col.shape[1])).contiguous()


def _attention_fwd(q, k, v, *, causal, scale=None, layout="bshd", return_lse=False, out=None, **kw):
    assert layout == "bshd" and not kw
    o, lse = O.attention(q, k, v, causal=causal, scale=scale)
    o = o.to(q.dtype)
    if out is not None:
        out.copy_(o)
        o = out
    return (o, lse) if return_lse else o


def _attention_bwd(d_out, q, k, v, out, lse, *, causal, scale=None, dq=None, dk=None, dv=None, **kw):
    calls["attention_bwd"] += 1
    assert not kw
    with torch.enable_grad():
        gq, gk, gv = O.attention_grads(q, k, v, d_out, causal=causal, scale=scale)
    if dq is None:
        return gq.to(q.dtype), gk.to(k.dtype), gv.to(v.dtype)
    dq.copy_(gq)
    dk.copy_(gk)
    dv.copy_(gv)
    return dq, dk, dv


SUBSTITUTES = {
    "linear": _linear,
    "layernorm": _layernorm,
    "layernorm_bwd": _layernorm_bwd,
    "bias_gelu": _bias_gelu,
    "gelu_bwd": _gelu_bwd,
    "ls_residual": _ls_residual,
    "ls_residual_bwd": _ls_residual_bwd,
    "pixel_shuffle": hostlogic.SUBSTITUTES["pixel_shuffle"],
    "pixel_shuffle_bwd": _pixel_shuffle_bwd,
    "patch_embed": _patch_embed,
    "patch_im2col": _patch_im2col,
    "attention_fwd": _attention_fwd,
    "attention_bwd": _attention_bwd,
}


@contextlib.contextmanager
def vision_oracle_ops():
    """hostlogic.oracle_ops() with the vision substitutes above (see module doc); resets `calls`."""
    from long_vita_b200 import ops

    calls.clear()
    saved = {name: getattr(ops, name) for name in SUBSTITUTES}
    with hostlogic.oracle_ops():
        try:
            for name, fn in SUBSTITUTES.items():
                setattr(ops, name, fn)
            yield ops
        finally:
            for name, fn in saved.items():
                setattr(ops, name, fn)
