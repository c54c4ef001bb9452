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

Megatron's `--use-kv-cache` generation (text_generation/generation.py:127-131: the prompt once, then one token per
forward) passes `inference_params` (megatron-core 0.7 `InferenceParams`).  The layers then share one K/V cache per
model, `key_value_memory_dict["b200_kv_cache"]`, made by the first layer of the first forward with
`hf.modeling.new_cache` (on the device, or partly in pinned host memory when it does not fit), exactly as the
Megatron-free `B200GPTVLModel` makes it.  Layer `layer_number` reads and writes its index `layer_number - 1`; the
cache's length follows `sequence_len_offset` (kv_cache's `commit_to`), and RoPE takes the rows [offset, offset + s)
of the `max_sequence_length`-row table Megatron passes.  The host tier's format is `config.kv_host_dtype` (absent:
bf16; torch.float8_e4m3fn is the lossy FP8 one).

FP8 (`--fp8-format e4m3|hybrid`, `config.fp8` = "e4m3" / "hybrid"; opt-in, lossy): every forward runs the four linears
(linear_qkv, linear_proj, linear_fc1, linear_fc2) in FP8, as TransformerEngine's fp8_autocast does around the
reference's layers.  Inference and `--use-kv-cache` decode use `DecoderLayer(linear_dtype=torch.float8_e4m3fn)`;
`_forward_train` uses `ops.linear_fp8_autograd`, with e4m3 gradients for "e4m3" and e5m2 gradients for "hybrid", and
dW in bf16 when `config.fp8_wgrad` is False.  Attention, the norms, RoPE, SwiGLU and the fp32 `main_grad` stay bf16 /
fp32.  Scales are current scales, computed from the tensor being quantised, so TransformerEngine's delayed-scaling
fields (fp8_margin, fp8_interval, fp8_amax_history_len, fp8_amax_compute_algo) have nothing to act on and are ignored.
fp8_dot_product_attention / fp8_multi_head_attention are refused (NotImplementedError), any other `fp8` value is a
ValueError, both when the layer is built.  `config.fp8` absent or None: the bf16 layer, unchanged.
"""
from __future__ import annotations

import types
from functools import partial
from typing import Optional

import torch

from .. import kv_cache, ops
from ..hf.modeling import PACKED_WITH_CACHE, DecoderLayer, attention_step, new_cache
from .core_attention import megatron_cp_context, megatron_cu_seqlens, megatron_packed_ends, records_grad


# config.fp8 (Megatron's --fp8-format) -> the format of the gradients in the FP8 backward products
FP8_GRAD_DTYPE = {"e4m3": torch.float8_e4m3fn, "hybrid": torch.float8_e5m2}


def _linear_fp8(x, weight, bias, accumulate_wgrad, *, grad_dtype, fp8_wgrad):
    return ops.linear_fp8_autograd(x, weight, bias, grad_dtype, fp8_wgrad, accumulate_wgrad)


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
        # the inference layer (hf.modeling.DecoderLayer) on re-ordered copies, rebuilt whenever a parameter changes
        self._decoder = None
        self._decoder_stamp = None
        self._dims = types.SimpleNamespace(num_attention_heads=np_, num_key_value_heads=ng, head_dim=hn,
                                           rms_norm_eps=self.eps, hidden_size=h, intermediate_size=ffn)
        self._rope_cache = (None, None, None)
        if int(getattr(config, "tensor_model_parallel_size", 1) or 1) > 1:
            raise NotImplementedError("B200TransformerLayer holds whole weights: tensor_model_parallel_size must be 1 "
                                      "(14B bf16 fits one 80 GB H100; the BASELINE configs are CP x DP)")
        self.cp_size = int(getattr(config, "context_parallel_size", 1) or 1)
        self._cp_ctx = None
        self.cp_group = getattr(config, "cp_group", None)   # tests / Megatron-free callers may hand the group in
        # the format of the host tier of a K/V cache this layer creates under inference_params (kv_cache.make_cache)
        self.kv_host_dtype = kv_cache.check_host_dtype(getattr(config, "kv_host_dtype", torch.bfloat16))
        self.fp8 = getattr(config, "fp8", None)
        if self.fp8 is not None:
            if self.fp8 not in FP8_GRAD_DTYPE:
                raise ValueError(f"config.fp8 must be None, 'e4m3' or 'hybrid', got {self.fp8!r}")
            for name in ("fp8_dot_product_attention", "fp8_multi_head_attention"):
                if getattr(config, name, False):
                    raise NotImplementedError(f"config.{name}: attention runs in bf16 under config.fp8 (only the "
                                              "linears are FP8)")
        self.fp8_wgrad = bool(getattr(config, "fp8_wgrad", True))
        # (parameter dict, name) of every parameter, for the stamp of _decoder_layer: looked up per call, so a
        # re-assigned parameter is seen, without walking the submodules on every forward
        self._param_slots = [(m._parameters, n) for m in self.modules() for n in m._parameters]

    def _decoder_layer(self) -> DecoderLayer:
        """The inference layer on this module's parameters: Megatron's grouped QKV rows [ng, (np/ng + 2), hn, h] become
        [all q | all k | all v] and fc1 = cat(gate, up) the interleaved SwiGLU operand.  The copies follow
        load_state_dict() / optimizer steps / .to(): every in-place update of a parameter bumps its `_version`, and a
        re-assigned `.data` or parameter changes `data_ptr()`."""
        stamp = tuple((d[n]._version, d[n].data_ptr()) for d, n in self._param_slots)
        if self._decoder is None or stamp != self._decoder_stamp:
            self._decoder = None               # free the stale copies before the new ones are made
            ng, hn, g = self.ng, self.hn, self.np // self.ng
            a, m = self.self_attention, self.mlp
            w = a.linear_qkv.weight.data.view(ng, g + 2, hn, -1)
            b = a.linear_qkv.bias.data.view(ng, g + 2, hn)
            fc1 = m.linear_fc1.weight.data
            p = "model.layers.0."
            hf = {p + "self_attn.o_proj.weight": a.linear_proj.weight.data,
                  p + "mlp.gate_proj.weight": fc1[: self.ffn], p + "mlp.up_proj.weight": fc1[self.ffn :],
                  p + "mlp.down_proj.weight": m.linear_fc2.weight.data,
                  p + "input_layernorm.weight": a.linear_qkv.layer_norm_weight.data,
                  p + "post_attention_layernorm.weight": m.linear_fc1.layer_norm_weight.data}
            for name, rows in (("q_proj", slice(0, g)), ("k_proj", g), ("v_proj", g + 1)):
                hf[p + f"self_attn.{name}.weight"] = w[:, rows].reshape(-1, w.shape[-1])
                hf[p + f"self_attn.{name}.bias"] = b[:, rows].reshape(-1)
            dtype = torch.bfloat16 if self.fp8 is None else torch.float8_e4m3fn
            self._decoder, self._decoder_stamp = DecoderLayer(self._dims, hf, 0, dtype), stamp
        return self._decoder

    def _cp(self, s: int, device):
        self._cp_ctx = megatron_cp_context(self._cp_ctx, self.cp_size, s, self.np, self.ng, self.hn, device, self.cp_group)
        return self._cp_ctx

    def _rope(self, rotary_pos_emb, holder=None):
        """Megatron hands the layer `freqs` [s, 1, 1, hn] fp32 (rotary_pos_embedding.py:84-122); the
        cos / sin tables (bf16, cast as at :200-201) are cached per tensor, in this layer or, under inference_params,
        in `holder` (the key_value_memory_dict the layers share: Megatron builds one table per forward for all of
        them)."""
        if isinstance(rotary_pos_emb, (tuple, list)):
            rotary_pos_emb = rotary_pos_emb[0]
        key, cos, sin = self._rope_cache if holder is None else holder.get("b200_rope", (None, None, None))
        if key is not rotary_pos_emb:
            f = rotary_pos_emb.reshape(rotary_pos_emb.shape[0], -1).float()
            cos, sin = torch.cos(f).to(torch.bfloat16), torch.sin(f).to(torch.bfloat16)
            if holder is None:
                self._rope_cache = (rotary_pos_emb, cos, sin)
            else:
                holder["b200_rope"] = (rotary_pos_emb, cos, sin)
        return cos, sin

    def forward(self, hidden_states, attention_mask=None, context=None, context_mask=None, rotary_pos_emb=None,
                inference_params=None, packed_seq_params=None):
        assert packed_seq_params is None, "Packed sequence is not supported by B200TransformerLayer."
        s, b, h = hidden_states.shape
        if b != 1:
            raise NotImplementedError("micro-batch 1 (the reference's long-context setting)")
        if inference_params is not None:
            return self._forward_cached(hidden_states, rotary_pos_emb, inference_params), context
        if records_grad(hidden_states, *self.parameters()):
            return self._forward_train(hidden_states, rotary_pos_emb), context
        layer = self._decoder_layer()
        cos, sin = (None, None) if rotary_pos_emb is None else self._rope(rotary_pos_emb)
        cp_ctx = self._cp(s, hidden_states.device)
        if cp_ctx is not None:
            attend = cp_ctx.attention_separate                                     # [s, np * hn]
        else:
            attend = partial(attention_step(cu_seqlens=megatron_cu_seqlens(s, hidden_states.device)), 0)
        x, d = layer.forward(hidden_states.reshape(s, h), None, cos, sin, attend)
        # plain residual add (bias-dropout-add with p = 0, no bias); a layer run in row chunks has added it already
        out = x if d is None else ops.ls_residual(x, d)
        return out.view(s, b, h), context

    def _forward_cached(self, hidden_states, rotary_pos_emb, ip):
        """forward() under Megatron's `--use-kv-cache` protocol (see the module doc).  Every refusal is raised before
        anything is launched."""
        s, b, h = hidden_states.shape
        if torch.is_grad_enabled() and records_grad(hidden_states, *self.parameters()):
            raise NotImplementedError("inference_params (the K/V cache of generation) with gradients enabled: "
                                      "training runs without it")
        if self.cp_size > 1:
            raise NotImplementedError("inference_params (--use-kv-cache) under context parallelism is not supported: "
                                      "the sharded cache lives in cp.ContextParallelRunner")
        if int(getattr(ip, "max_batch_size", 1) or 1) > 1:
            raise NotImplementedError(f"inference_params.max_batch_size {ip.max_batch_size}: the K/V cache holds one "
                                      "sequence (micro-batch 1)")
        if megatron_packed_ends() is not None:
            raise NotImplementedError(PACKED_WITH_CACHE)
        offset = int(ip.sequence_len_offset)
        if rotary_pos_emb is not None:
            rows = (rotary_pos_emb[0] if isinstance(rotary_pos_emb, (tuple, list)) else rotary_pos_emb).shape[0]
            if rows < offset + s:
                raise ValueError(f"rotary_pos_emb has {rows} rows; the tokens at sequence_len_offset {offset} need "
                                 f"{offset + s} (Megatron builds it for max_sequence_length positions)")
        kv = ip.key_value_memory_dict
        cache = kv.get("b200_kv_cache")
        if cache is None:
            capacity = int(getattr(ip, "max_sequence_length", 0) or (s + 1024))
            cache = new_cache(self._dims, int(self.config.num_layers), capacity, s, hidden_states.device,
                              self.kv_host_dtype)
            kv["b200_kv_cache"] = cache
        cache.commit_to(offset)
        attend = partial(attention_step(cache, None, s), self.layer_number - 1)
        layer = self._decoder_layer()
        cos = sin = None
        if rotary_pos_emb is not None:
            cos, sin = self._rope(rotary_pos_emb, kv)
            cos, sin = cos[offset : offset + s], sin[offset : offset + s]             # views: no table per layer
        x, d = layer.forward(hidden_states.reshape(s, h), None, cos, sin, attend)
        out = x if d is None else ops.ls_residual(x, d)
        return out.view(s, b, h)

    # -- training: the same layer out of differentiable pieces (ops.*_autograd) --------------------------------
    def _forward_train(self, hidden_states, rotary_pos_emb):
        """Forward that records an autograd graph: every operator is a torch.autograd.Function over the C-ABI kernels
        (RMSNorm / SwiGLU / RoPE backward kernels, `lv_attn_bwd`, and the wgmma GEMM for dX and dW).  It works on the
        Megatron parameter layouts directly (grouped QKV rows, fc1 = cat(gate, up)), so gradients land on the
        parameters Megatron's optimizer owns; the fused-epilogue / in-place shortcuts of the inference path are not
        used here (the un-fused gate|up activation is what the SwiGLU backward needs).

        `config.gradient_accumulation_fusion` (absent: off) adds the four weight gradients to each weight's fp32
        `main_grad` inside the GEMM, as Megatron's linears do (ops.linear_autograd, accumulate_wgrad).

        With `config.fp8` the four linears are ops.linear_fp8_autograd (see the module doc); nothing else changes."""
        s, b, h = hidden_states.shape
        np_, ng, hn = self.np, self.ng, self.hn
        g = np_ // ng
        self._decoder = None               # the re-ordered inference copies go stale once the parameters train
        fuse = bool(getattr(self.config, "gradient_accumulation_fusion", False))
        linear = ops.linear_autograd
        if self.fp8 is not None:
            # the weights are quantised by every forward (W) and backward (W^T), from their current values: Megatron's
            # optimizers write updated weights into .data, which moves neither _version nor data_ptr
            linear = partial(_linear_fp8, grad_dtype=FP8_GRAD_DTYPE[self.fp8], fp8_wgrad=self.fp8_wgrad)
        x = hidden_states.reshape(s, h)
        a = self.self_attention
        hcur = ops.rmsnorm_autograd(x, a.linear_qkv.layer_norm_weight, self.eps)
        qkv = linear(hcur, a.linear_qkv.weight, a.linear_qkv.bias, fuse).view(s, ng, g + 2, hn)
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
        o = linear(att.reshape(s, np_ * hn), a.linear_proj.weight, None, fuse)
        hcur, x = ops.rmsnorm_autograd(o, self.mlp.linear_fc1.layer_norm_weight, self.eps, residual=x)
        gate_up = linear(hcur, self.mlp.linear_fc1.weight, None, fuse)             # cat(gate, up)
        d = linear(ops.swiglu_autograd(gate_up), self.mlp.linear_fc2.weight, None, fuse)
        return (x + d).view(s, b, h)


def get_b200_layer_spec():
    """`--spec long_vita_b200.megatron.transformer_layer get_b200_layer_spec`."""
    try:
        from megatron.core.transformer.spec_utils import ModuleSpec
    except ImportError:   # Megatron is un-vendored in the build container: same dataclass shape
        from .stub import ModuleSpec
    return ModuleSpec(module=B200TransformerLayer)
