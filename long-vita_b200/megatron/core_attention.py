"""Megatron-core operator surface of the attention hot path (SURVEY.md 8b, boundaries B1 and B3).

B1 - `B200DotProductAttention`: a `core_attention` module with the constructor / forward the
reference's layer specs expect (long_vita_megatron/core/models/gpt/gpt_layer_specs.py:38-44 puts
`TEDotProductAttention` there; vit_layer_specs.py:87-91 the ViT twin).  Megatron 0.7 builds it as
`cls(config, layer_number, attn_mask_type, attention_type)` and calls
`forward(query, key, value, attention_mask, attn_mask_type=, packed_seq_params=)` with
query [sq, b, np, hn], key/value [sk, b, ng, hn] (GQA not expanded) and expects [sq, b, np*hn]
(long_vita_megatron/core/transformer/dot_product_attention.py:153, 176-184, 392).

B3 - `b200_dot_product_attention_forward_wrapper`: a function whose name ends in `wrapper`, so the
reference's patch registry treats it as a decorator over the original
`DotProductAttention.forward` (patch_utils.py:46-53, 62-63):
    MindSpeedPatchesManager.register_patch(
        'megatron.core.transformer.dot_product_attention.DotProductAttention.forward',
        b200_dot_product_attention_forward_wrapper)
registered after `import long_vita_megatron.megatron_adaptor` (megatron_adaptor.py:21-22).

Megatron-core is NOT importable in the build container (un-vendored submodule, SURVEY.md fact 2), so
nothing here imports it: the mask type is duck-typed by name and process-group lookups go through
`parallel_state` only when context parallelism is on.

Packed samples (`--reset-position-ids --reset-attention-mask`, every shipped fine-tuning script): the data pipeline
concatenates samples into one row and the training loop publishes the sample ends through
`long_vita_megatron.training.utils.set_actual_seq_len` (training/utils.py:509-511; only set under
`--reset-attention-mask`).  When that list has more than one entry, attention is causal inside each sample and blind
across samples (lv_attn_docs_fwd / lv_attn_docs_bwd), the mask of get_ltor_masks_and_position_ids
(training/utils.py:192-249).  tests/test_gpu_surfaces.py (kernels) and
tests/test_surfaces_host.py (host logic, CPU) drive these objects with a stub that reproduces the
ModuleSpec / build_module calling convention.
"""
from __future__ import annotations

import math
import sys
from functools import wraps
from typing import Optional

import torch

from .. import ops


def _is_causal(attn_mask_type) -> bool:
    """AttnMaskType.causal / padding_causal -> True; no_mask / padding -> False (duck-typed by name)."""
    name = getattr(attn_mask_type, "name", str(attn_mask_type)).lower()
    return "causal" in name


_CU_CACHE = [None, None]   # (sample ends, device) -> cu_seqlens tensor of the current micro-batch


def megatron_packed_ends():
    """The sample ends of this micro-batch's packed row inside a Megatron job (`get_actual_seq_len()` of the reference's
    training utils), or None: no Megatron job, no --reset-attention-mask, or a single sample."""
    utils = sys.modules.get("long_vita_megatron.training.utils")   # imported by the training loop that publishes it
    if utils is None or not hasattr(utils, "get_actual_seq_len"):
        return None
    ends = utils.get_actual_seq_len()
    return None if ends is None or len(ends) <= 1 else ends


def megatron_cu_seqlens(seq_len: int, device) -> Optional[torch.Tensor]:
    """cu_seqlens of the packed row of this micro-batch (None if it is not packed).  The int32 device copy is made once
    per micro-batch (when the list changes) and shared by every layer."""
    ends = megatron_packed_ends()
    if ends is None:
        return None
    key = (tuple(int(e) for e in ends), str(device), int(seq_len))
    if _CU_CACHE[0] != key:
        _CU_CACHE[0], _CU_CACHE[1] = key, ops.packed_cu_seqlens(actual_seq_len=list(key[0]), device=device,
                                                                 seq_len=seq_len)
    return _CU_CACHE[1]


def megatron_cp_context(cached, cp_size: int, seq_len: int, hq: int, hkv: int, hn: int, device, group=None):
    """Context parallelism (zig-zag shards, training/utils.py:329-341): a layer receives this rank's `seq_len` rows
    only, so attention must see the other ranks' K/V - `cp.CPContext` (fused in-kernel exchange forward, all-gather /
    reduce-scatter backward).  Returns `cached` while it fits this length (a micro-batch of another length gets its own
    buffers), None when context_parallel_size is 1.  `group` defaults to Megatron's context-parallel group."""
    if cp_size <= 1:
        return None
    if megatron_packed_ends() is not None:
        raise NotImplementedError("packed samples (--reset-attention-mask) under context parallelism are not supported")
    if cached is not None and cached.S == seq_len * cp_size:
        return cached
    from ..cp import CPContext

    if group is None:
        from megatron.core import parallel_state as mpu   # only reached inside a Megatron job

        group = mpu.get_context_parallel_group()
    return CPContext.shared(group, seq_len * cp_size, hq, hkv, hn, device, fused_qkv=False)


def records_grad(*ts) -> bool:
    """Training or inference: an autograd graph is recorded when gradients are enabled and an input needs one."""
    return torch.is_grad_enabled() and any(t.requires_grad for t in ts)


def _attention_sbhd(query, key, value, causal: bool, scale: float, cp_ctx=None, cu_seqlens=None):
    sq, b, np_, hn = query.shape
    if cu_seqlens is not None:
        if cp_ctx is not None:
            raise NotImplementedError("packed samples (--reset-attention-mask) under context parallelism are not supported")
        if not causal:
            raise NotImplementedError("packed samples need a causal attention mask")
        if b != 1:
            raise NotImplementedError("packed samples need micro-batch 1")
    train = records_grad(query, key, value)
    if cp_ctx is not None:
        if b != 1:
            raise AssertionError("context-parallel attention supports micro-batch 1 (the reference's long-context setting)")
        if train:
            from ..cp import cp_attention      # training: fused exchange forward + lv_attn_bwd / reduce-scatter backward

            out = cp_attention(query[:, 0], key[:, 0], value[:, 0], cp_ctx, scale)
        else:
            out = cp_ctx.attention_separate(query[:, 0], key[:, 0], value[:, 0], scale=scale)   # [sq, np*hn]
        return out.view(sq, 1, np_ * hn)
    docs = ops.docs_kwargs(cu_seqlens)
    if train:
        # training: differentiable path (lv_attn_bwd through torch.autograd.Function)
        out = ops.attention(query.permute(1, 0, 2, 3), key.permute(1, 0, 2, 3), value.permute(1, 0, 2, 3),
                            causal=causal, scale=scale, **docs)                # [b, sq, np, hn]
        return out.permute(1, 0, 2, 3).reshape(sq, b, np_ * hn)
    out = ops.attention_fwd(query, key, value, causal=causal, scale=scale, layout="sbhd", **docs)
    return out.reshape(sq, b, np_ * hn)


class B200DotProductAttention(torch.nn.Module):
    """Drop-in for the `core_attention` ModuleSpec slot."""

    def __init__(self, config, layer_number: int, attn_mask_type, attention_type: str = "self",
                 attention_dropout: Optional[float] = None):
        super().__init__()
        self.config = config
        self.layer_number = max(1, layer_number)
        self.attn_mask_type = attn_mask_type
        self.attention_type = attention_type
        p = config.attention_dropout if attention_dropout is None else attention_dropout
        if p not in (0, 0.0, None):
            raise ValueError("attention dropout is not supported by the fused kernel (the reference trains with 0.0)")
        kv_channels = getattr(config, "kv_channels", None) or config.hidden_size // config.num_attention_heads
        self.hidden_size_per_attention_head = kv_channels
        self.softmax_scale = 1.0 / math.sqrt(kv_channels)
        if getattr(config, "apply_query_key_layer_scaling", False):
            # Megatron divides by layer_number and multiplies back inside the fp32 softmax: a no-op here
            pass
        self.cp_size = int(getattr(config, "context_parallel_size", 1) or 1)
        self._cp_ctx = None

    def forward(self, query, key, value, attention_mask=None, attn_mask_type=None, packed_seq_params=None):
        assert packed_seq_params is None, (
            "Packed sequence is not supported by B200DotProductAttention."     # same contract as the reference,
        )                                                                     # dot_product_attention.py:156-159
        mask_type = self.attn_mask_type if attn_mask_type is None else attn_mask_type
        causal = _is_causal(mask_type)
        cp_ctx = None
        if _is_causal(self.attn_mask_type):
            sq, _, np_, hn = query.shape
            cp_ctx = self._cp_ctx = megatron_cp_context(self._cp_ctx, self.cp_size, sq, np_, key.shape[2], hn,
                                                        query.device)
        cu = None if cp_ctx is not None else megatron_cu_seqlens(query.shape[0], query.device)
        return _attention_sbhd(query, key, value, causal, self.softmax_scale, cp_ctx, cu)


def b200_dot_product_attention_forward_wrapper(fn):
    """Decorator-style patch for `DotProductAttention.forward` (see module docstring)."""

    @wraps(fn)
    def wrapper(self, query, key, value, attention_mask, attn_mask_type=None, packed_seq_params=None):
        assert packed_seq_params is None, (
            "Packed sequence is not supported by DotProductAttention."
            "Please use TEDotProductAttention instead."
        )
        if not (query.is_cuda and query.dtype == torch.bfloat16):
            return fn(self, query, key, value, attention_mask, attn_mask_type, packed_seq_params)
        mask_type = getattr(self, "attn_mask_type", None) if attn_mask_type is None else attn_mask_type
        hn = query.shape[-1]
        scale = getattr(self, "softmax_scale", None) or 1.0 / math.sqrt(hn)
        return _attention_sbhd(query, key, value, _is_causal(mask_type), scale,
                               cu_seqlens=megatron_cu_seqlens(query.shape[0], query.device))

    return wrapper


def b200_gpt_vl_model_init_wrapper(orig_init):
    """Decorates `GPTVLModel.__init__` (long_vita_megatron/core/models/multimodal/gpt_vl_model.py:72-114) so that the
    reference's stock `vision_model_provider` (pretrain_long_vita.py:599-601, handed over as
    `external_feature_model_provider` at :641-655) is replaced by `b200_vision_model_provider` at the moment the model
    is built.  Patching the class rather than the provider's module-level name works however the training script is
    started: `torchrun pretrain_long_vita.py` runs it as `__main__`, whose own copy of the function `model_provider`
    passes, and a second import of `long_vita_megatron.pretrain_long_vita` would be a different function object.
    Any other provider (a caller's own, or None) is passed through unchanged."""
    from .vision_model import b200_vision_model_provider

    @wraps(orig_init)
    def __init__(self, *args, **kwargs):
        prov = kwargs.get("external_feature_model_provider")
        if prov is not None and getattr(prov, "__name__", "") == "vision_model_provider":
            kwargs["external_feature_model_provider"] = b200_vision_model_provider
        return orig_init(self, *args, **kwargs)

    return __init__


def register_b200_patches(patches_manager=None, vision_model: bool = False) -> None:
    """Register + apply the attention patch through the reference's own registry
    (long_vita_megatron/patch_utils.py:105-118).  Call after importing
    long_vita_megatron.megatron_adaptor.

    `vision_model=True` also builds the vision side (InternViT-300M + projector) as `B200VisionModel`, forward and
    backward on the fused kernels (`b200_gpt_vl_model_init_wrapper`).  It is opt-in: the provider refuses
    configurations it does not implement (tensor parallelism > 1, recompute, vision context parallelism, other towers).
    With the whole tower trained a step is still slower than the stock modules: 477 ms against 389 ms for eager bf16
    PyTorch at 64 frames on one H100 80GB HBM3 at 700 W (DESIGN.md §8)."""
    if patches_manager is None:
        from long_vita_megatron.patch_utils import MindSpeedPatchesManager as patches_manager  # noqa: N813
    patches_manager.register_patch(
        "megatron.core.transformer.dot_product_attention.DotProductAttention.forward",
        b200_dot_product_attention_forward_wrapper,
    )
    if vision_model:
        patches_manager.register_patch("long_vita_megatron.core.models.multimodal.gpt_vl_model.GPTVLModel.__init__",
                                       b200_gpt_vl_model_init_wrapper)
    patches_manager.apply_patches()
