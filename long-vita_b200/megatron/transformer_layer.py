"""Whole-layer `--spec` module (SURVEY.md 8b, boundary B2).

`pretrain_long_vita.py:631-632` / `run_text_generation_server.py:57-58` load
`transformer_layer_spec = import_module(args.spec)`; `get_b200_layer_spec()` returns a
`ModuleSpec(module=B200TransformerLayer)` for it.  The layer is called the way
long_vita_megatron/core/transformer/transformer_block.py:232-240 calls it,
    layer(hidden_states=, attention_mask=, context=, context_mask=, rotary_pos_emb=,
          inference_params=, packed_seq_params=)  ->  (hidden_states, context)
with hidden_states [s, b, h] (transformer_layer.py:173-182, 257), and runs the fused hot path:
RMSNorm (+ fused residual add) -> QKV GEMM + bias -> RoPE in place -> fused attention ->
O-proj GEMM -> RMSNorm + add -> gate|up GEMM -> SwiGLU -> down GEMM.

State-dict names are TransformerEngine's, so Megatron checkpoints load unchanged
(long_vita_megatron/ckpt_convert_modellink_to_megatron_with_te.py:36-41,
tools/hf2mcore_long_vita.py:486-507):
    self_attention.linear_qkv.layer_norm_weight | .weight | .bias
    self_attention.linear_proj.weight
    mlp.linear_fc1.layer_norm_weight | .weight          (fc1 = cat(gate, up))
    mlp.linear_fc2.weight
`linear_qkv.weight` is in Megatron's grouped layout [ng, (np/ng + 2), hn, h] (q heads of a group,
then its k, then its v; hf2mcore_long_vita.py:488-498); it is re-ordered once, lazily, into
[all q | all k | all v] so that q/k/v are uniformly strided views of one GEMM output.

Packed samples (`--reset-attention-mask`): when the training loop has published more than one sample end through
`long_vita_megatron.training.utils.set_actual_seq_len`, attention is causal within each sample only
(core_attention.megatron_cu_seqlens; lv_attn_docs_fwd / lv_attn_docs_bwd).  Not combined with context parallelism.

Inference takes the fused path (GEMM epilogues, in-place RoPE, fused add + norm).  When gradients are enabled and
anything requires grad, `_forward_train` builds the same layer from differentiable pieces whose backward passes are
kernels too (`lv_rmsnorm_bwd`, `lv_swiglu_bwd`, `lv_attn_bwd`, the GEMM on transposed operands).
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import ops
from .core_attention import megatron_cu_seqlens, megatron_packed_ends


class _Params(torch.nn.Module):
    """Empty container so parameters get TE's dotted names."""


class B200TransformerLayer(torch.nn.Module):
    def __init__(self, config, submodules=None, layer_number: int = 1, hidden_dropout: Optional[float] = None):
        super().__init__()
        self.config = config
        self.layer_number = layer_number
        h = config.hidden_size
        np_ = config.num_attention_heads
        ng = getattr(config, "num_query_groups", None) or np_
        hn = getattr(config, "kv_channels", None) or h // np_
        ffn = config.ffn_hidden_size
        if getattr(config, "hidden_dropout", 0.0) not in (0, 0.0) or getattr(config, "attention_dropout", 0.0) not in (0, 0.0):
            raise ValueError("dropout is not supported on the fused path (the reference trains with 0.0)")
        self.np, self.ng, self.hn, self.ffn = np_, ng, hn, ffn
        self.eps = getattr(config, "layernorm_epsilon", 1e-6)
        dt = getattr(config, "params_dtype", torch.bfloat16)
        dev = torch.cuda.current_device() if torch.cuda.is_available() else "cpu"

        def P(*shape, ones=False):
            t = torch.ones(*shape, dtype=dt, device=dev) if ones else torch.empty(*shape, dtype=dt, device=dev).normal_(0, 0.02)
            return torch.nn.Parameter(t, requires_grad=False)

        self.self_attention = _Params()
        self.self_attention.linear_qkv = _Params()
        self.self_attention.linear_qkv.layer_norm_weight = P(h, ones=True)
        self.self_attention.linear_qkv.weight = P((np_ + 2 * ng) * hn, h)
        self.self_attention.linear_qkv.bias = torch.nn.Parameter(torch.zeros((np_ + 2 * ng) * hn, dtype=dt, device=dev),
                                                               requires_grad=False)
        self.self_attention.linear_proj = _Params()
        self.self_attention.linear_proj.weight = P(h, np_ * hn)
        self.mlp = _Params()
        self.mlp.linear_fc1 = _Params()
        self.mlp.linear_fc1.layer_norm_weight = P(h, ones=True)
        self.mlp.linear_fc1.weight = P(2 * ffn, h)
        self.mlp.linear_fc2 = _Params()
        self.mlp.linear_fc2.weight = P(h, ffn)
        self._qkv_w = None       # re-ordered copies of the parameters, rebuilt whenever a parameter changes
        self._qkv_b = None
        self._fused_versions = None
        self._rope_cache = (None, None, None)
        if int(getattr(config, "tensor_model_parallel_size", 1) or 1) > 1:
            raise NotImplementedError("B200TransformerLayer holds whole weights: tensor_model_parallel_size must be 1 "
                                      "(14B bf16 fits one 80 GB H100; the BASELINE configs are CP x DP)")
        self.cp_size = int(getattr(config, "context_parallel_size", 1) or 1)
        self._cp_ctx = None
        self.cp_group = getattr(config, "cp_group", None)   # tests / Megatron-free callers may hand the group in

    # -- Megatron grouped QKV rows -> [q | k | v] -------------------------------------------------
    def _ungroup(self):
        np_, ng, hn = self.np, self.ng, self.hn
        g = np_ // ng
        w = self.self_attention.linear_qkv.weight.data.view(ng, g + 2, hn, -1)
        b = self.self_attention.linear_qkv.bias.data.view(ng, g + 2, hn)
        self._qkv_w = torch.cat([w[:, :g].reshape(np_ * hn, -1), w[:, g].reshape(ng * hn, -1),
                                 w[:, g + 1].reshape(ng * hn, -1)], dim=0).contiguous()
        self._qkv_b = torch.cat([b[:, :g].reshape(-1), b[:, g].reshape(-1), b[:, g + 1].reshape(-1)]).contiguous()
        fc1 = self.mlp.linear_fc1.weight.data                      # cat(gate, up) -> rows (gate_i, up_i)
        self._fc1_w = ops.interleave_gate_up(fc1[: self.ffn], fc1[self.ffn :])

    def _fused_weights_current(self) -> bool:
        """The re-ordered copies follow load_state_dict() / optimizer steps: every in-place update of a parameter bumps
        its `_version`, and a re-assigned `.data` changes `data_ptr()`."""
        ps = (self.self_attention.linear_qkv.weight, self.self_attention.linear_qkv.bias, self.mlp.linear_fc1.weight)
        stamp = tuple((p._version, p.data_ptr()) for p in ps)
        if self._qkv_w is None or stamp != self._fused_versions:
            self._ungroup()
            self._fused_versions = stamp
        return True

    def _cp(self, s: int, device):
        """Context parallelism (zig-zag shards, training/utils.py:329-341): the layer receives this rank's rows only,
        so attention must see the other ranks' K/V - `cp.CPContext` (fused in-kernel exchange forward, all-gather /
        reduce-scatter backward).  None when context_parallel_size == 1."""
        if self.cp_size <= 1:
            return None
        if megatron_packed_ends() is not None:
            raise NotImplementedError("packed samples (--reset-attention-mask) under context parallelism are not supported")
        if self._cp_ctx is None or self._cp_ctx.S != s * self.cp_size:
            from ..cp import CPContext

            group = self.cp_group
            if group is None:
                from megatron.core import parallel_state as mpu   # only reached inside a Megatron job

                group = mpu.get_context_parallel_group()
            self._cp_ctx = CPContext.shared(group, s * self.cp_size, self.np, self.ng, self.hn, device, fused_qkv=False)
        return self._cp_ctx

    def _rope(self, rotary_pos_emb):
        """Megatron hands the layer `freqs` [s, 1, 1, hn] fp32 (rotary_pos_embedding.py:84-122); the
        cos / sin tables (bf16, cast as at :200-201) are cached per tensor."""
        if isinstance(rotary_pos_emb, (tuple, list)):
            rotary_pos_emb = rotary_pos_emb[0]
        key, cos, sin = self._rope_cache
        if key is not rotary_pos_emb:
            f = rotary_pos_emb.reshape(rotary_pos_emb.shape[0], -1).float()
            cos, sin = torch.cos(f).to(torch.bfloat16), torch.sin(f).to(torch.bfloat16)
            self._rope_cache = (rotary_pos_emb, cos, sin)
        return cos, sin

    def forward(self, hidden_states, attention_mask=None, context=None, context_mask=None, rotary_pos_emb=None,
                inference_params=None, packed_seq_params=None):
        assert packed_seq_params is None, "Packed sequence is not supported by B200TransformerLayer."
        if inference_params is not None:
            raise NotImplementedError("KV-cache decode is outside this build's scope (prefill forward only)")
        s, b, h = hidden_states.shape
        if b != 1:
            raise NotImplementedError("micro-batch 1 (the reference's long-context setting)")
        if torch.is_grad_enabled() and (hidden_states.requires_grad or any(p.requires_grad for p in self.parameters())):
            return self._forward_train(hidden_states, rotary_pos_emb), context
        self._fused_weights_current()
        np_, ng, hn = self.np, self.ng, self.hn
        x = hidden_states.reshape(s, h)
        hcur = ops.rmsnorm(x, self.self_attention.linear_qkv.layer_norm_weight, self.eps)
        qkv = ops.linear(hcur, self._qkv_w, self._qkv_b)
        q = qkv[:, : np_ * hn].view(s, np_, hn)
        k = qkv[:, np_ * hn : (np_ + ng) * hn].view(s, ng, hn)
        v = qkv[:, (np_ + ng) * hn :].view(s, ng, hn)
        if rotary_pos_emb is not None:
            cos, sin = self._rope(rotary_pos_emb)
            ops.rope(q, cos, sin, out=q)
            ops.rope(k, cos, sin, out=k)
        cp_ctx = self._cp(s, hidden_states.device)
        if cp_ctx is not None:
            att = cp_ctx.attention_separate(q, k, v)                               # [s, np * hn]
        else:
            att = ops.attention_fwd(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0), causal=True,
                                    **ops.docs_kwargs(megatron_cu_seqlens(s, hidden_states.device)))
        o = ops.linear(att.view(s, np_ * hn), self.self_attention.linear_proj.weight)
        hcur, x = ops.rmsnorm(o, self.mlp.linear_fc1.layer_norm_weight, self.eps, residual=x)
        a = ops.linear(hcur, self._fc1_w, act="swiglu")
        d = ops.linear(a, self.mlp.linear_fc2.weight)
        out = ops.ls_residual(x, d)           # plain residual add (bias-dropout-add with p = 0, no bias)
        return out.view(s, b, h), context


    # -- training: the same layer out of differentiable pieces (ops.*_autograd) --------------------------------
    def _forward_train(self, hidden_states, rotary_pos_emb):
        """Forward that records an autograd graph: every operator is a torch.autograd.Function over the C-ABI kernels
        (RMSNorm / SwiGLU / RoPE backward kernels, `lv_attn_bwd`, and the wgmma GEMM for dX and dW).  It works on the
        Megatron parameter layouts directly (grouped QKV rows, fc1 = cat(gate, up)), so gradients land on the
        parameters Megatron's optimizer owns; the fused-epilogue / in-place shortcuts of the inference path are not
        used here (the un-fused gate|up activation is what the SwiGLU backward needs)."""
        s, b, h = hidden_states.shape
        np_, ng, hn = self.np, self.ng, self.hn
        g = np_ // ng
        self._qkv_w = None                 # the re-ordered inference copies go stale once the parameters train
        x = hidden_states.reshape(s, h)
        a = self.self_attention
        hcur = ops.rmsnorm_autograd(x, a.linear_qkv.layer_norm_weight, self.eps)
        qkv = ops.linear_autograd(hcur, a.linear_qkv.weight, a.linear_qkv.bias).view(s, ng, g + 2, hn)
        q = qkv[:, :, :g].reshape(s, np_, hn)
        k = qkv[:, :, g].contiguous()
        v = qkv[:, :, g + 1].contiguous()
        if rotary_pos_emb is not None:
            cos, sin = self._rope(rotary_pos_emb)
            q = ops.rope_autograd(q, cos, sin)
            k = ops.rope_autograd(k, cos, sin)
        cp_ctx = self._cp(s, hidden_states.device)
        if cp_ctx is not None:
            from ..cp import cp_attention

            att = cp_attention(q.contiguous(), k, v, cp_ctx)                                    # [s, np * hn]
        else:
            att = ops.attention(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0), causal=True,
                                **ops.docs_kwargs(megatron_cu_seqlens(s, hidden_states.device)))    # [1, s, np, hn]
        o = ops.linear_autograd(att.reshape(s, np_ * hn), a.linear_proj.weight)
        hcur, x = ops.rmsnorm_autograd(o, self.mlp.linear_fc1.layer_norm_weight, self.eps, residual=x)
        gate_up = ops.linear_autograd(hcur, self.mlp.linear_fc1.weight)                         # cat(gate, up)
        d = ops.linear_autograd(ops.swiglu_autograd(gate_up), self.mlp.linear_fc2.weight)
        return (x + d).view(s, b, h)


def get_b200_layer_spec():
    """`--spec long_vita_b200.megatron.transformer_layer get_b200_layer_spec`."""
    try:
        from megatron.core.transformer.spec_utils import ModuleSpec
    except ImportError:   # Megatron is un-vendored in the build container: same dataclass shape
        from .stub import ModuleSpec
    return ModuleSpec(module=B200TransformerLayer)
