"""HF-side attention boundary (SURVEY.md 8b, B4).

* `b200_attention_forward` has the signature transformers' `AttentionInterface` dispatches to
  (`ALL_ATTENTION_FUNCTIONS[name](module, query[b,h,s,d], key[b,hkv,s,d], value, attention_mask,
  dropout=, scaling=, **kw) -> (out[b,s,h,d], None)`); `register()` installs it under the name
  "b200_fa" so a stock HF Qwen2 / Long-VITA model runs on it with
  `attn_implementation="b200_fa"` where the reference passes "flash_attention_2"
  (tools/inference_long_vita.py:816).  Packed rows are honoured as transformers' `_flash_attention_forward` honours
  them: pre-computed `cu_seq_lens_q` / `cu_seq_lens_k` in the kwargs (equal: self-attention), or batch-1
  `position_ids` that are not one increasing run (its `_is_packed_sequence`), whose restarts at 0 are the document
  boundaries (`prepare_fa_kwargs_from_position_ids`).  Attention then stays inside each document (lv_attn_docs_fwd).
* `B200FlashAttention` replaces `InternAttention.inner_attn`
  (long_vita/models/long_vita_qwen2_intern/modeling_intern_vit.py:140-141, 173-175): same
  constructor and `forward(qkv[B,S,3,H,D], key_padding_mask=None, causal=False, ...)
  -> (out[B,S,H,D], None)` contract and the same assertions as
  long_vita/models/long_vita_qwen2_intern/flash_attention.py:31-42.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import ops

NAME = "b200_fa"

_POS_CACHE = [None, None, None]   # (position_ids tensor, its version, cu_seqlens): one lookup per forward, not per layer


def _is_packed_sequence(position_ids, batch_size: int) -> bool:
    """transformers' rule (modeling_flash_attention_utils._is_packed_sequence): batch 1 and the positions are not
    `arange(s) + min`."""
    if position_ids is None or batch_size != 1:
        return False
    ramp = torch.arange(position_ids.shape[-1], device=position_ids.device) + position_ids.min()
    return bool((ramp - position_ids).abs().sum())


def _packed_cu_seqlens(query, kwargs):
    cu_q, cu_k = kwargs.get("cu_seq_lens_q"), kwargs.get("cu_seq_lens_k")
    if cu_q is not None or cu_k is not None:
        if cu_q is None or cu_k is None or not torch.equal(cu_q, cu_k):
            raise NotImplementedError("b200_fa: packed rows need cu_seq_lens_q == cu_seq_lens_k (self-attention)")
        return cu_q.to(device=query.device, dtype=torch.int32).contiguous()
    pos = kwargs.get("position_ids")
    if pos is None:
        return None
    if _POS_CACHE[0] is pos and _POS_CACHE[1] == pos._version:
        return _POS_CACHE[2]
    cu = None
    if _is_packed_sequence(pos, query.shape[0]):
        cu = ops.packed_cu_seqlens(pos, device=query.device, seq_len=query.shape[2])
    _POS_CACHE[:] = [pos, pos._version, cu]
    return cu


def b200_attention_forward(module, query, key, value, attention_mask=None, dropout: float = 0.0,
                           scaling: Optional[float] = None, is_causal: Optional[bool] = None, **kwargs):
    if dropout:
        raise NotImplementedError("attention dropout is not supported by the fused kernel")
    if kwargs.get("sliding_window") not in (None, 0) and kwargs["sliding_window"] < key.shape[2]:
        raise NotImplementedError("sliding-window attention is not used by Long-VITA (use_sliding_window=false)")
    if attention_mask is not None:
        # The fused kernel applies the causal (or no) mask itself; any OTHER masking must be refused, not ignored.
        if attention_mask.dim() == 2:                       # [b, sk] key-padding mask (flash_attention_2 style)
            if not bool(attention_mask.to(torch.bool).all()):
                raise NotImplementedError("padding masks are not supported; pass unpadded sequences (batch 1)")
        elif attention_mask.dim() == 4:
            # [b, 1, sq, sk] masks transformers builds for sdpa / eager: bool (True = attend) or additive (0 = attend).
            # Pure causal <=> the LAST query row attends to every key (a padded key column would be masked there too).
            last = attention_mask[:, :, -1, :]
            visible = last if attention_mask.dtype == torch.bool else (last == 0)
            if not bool(visible.all()):
                raise NotImplementedError("b200_fa: the 4-D attention mask hides keys from the last query (padding or a "
                                          "custom mask); only pure causal / full attention on unpadded inputs is supported")
        else:
            raise NotImplementedError(f"b200_fa: unsupported attention_mask rank {attention_mask.dim()}")
    if is_causal is None:
        is_causal = bool(getattr(module, "is_causal", True)) and query.shape[2] > 1
    cu = _packed_cu_seqlens(query, kwargs)
    if cu is not None and not is_causal:
        raise NotImplementedError("b200_fa: packed rows without a causal mask are not supported")
    out = ops.attention_fwd(query, key, value, causal=is_causal, scale=scaling, layout="bhsd",
                            **ops.docs_kwargs(cu))                                                   # [b,h,s,d]
    return out.transpose(1, 2), None


def register(name: str = NAME) -> str:
    from transformers import AttentionInterface

    AttentionInterface.register(name, b200_attention_forward)
    return name


class B200FlashAttention(torch.nn.Module):
    def __init__(self, softmax_scale=None, attention_dropout=0.0, device=None, dtype=None):
        super().__init__()
        self.softmax_scale = softmax_scale
        self.dropout_p = attention_dropout

    def forward(self, qkv, key_padding_mask=None, causal=False, cu_seqlens=None, max_s=None, need_weights=False):
        assert not need_weights
        assert qkv.dtype in [torch.float16, torch.bfloat16]
        assert qkv.is_cuda
        if qkv.dtype != torch.bfloat16:
            raise NotImplementedError("B200FlashAttention computes in bfloat16 (the reference's torch_dtype)")
        if key_padding_mask is not None or cu_seqlens is not None:
            raise NotImplementedError("padded / packed inputs are not on the Long-VITA path (fixed 1025-token frames)")
        if self.training and self.dropout_p:
            raise NotImplementedError("attention dropout is not supported by the fused kernel")
        out = ops.attention_fwd(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], causal=causal, scale=self.softmax_scale)
        return out, None
