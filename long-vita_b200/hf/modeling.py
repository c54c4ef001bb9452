"""H100-native Long-VITA forward with the reference's HF `forward()` surface.

`LongVITAModel.forward` / `LongVITAForCausalLM.forward` keep the argument list of
long_vita/models/long_vita_qwen2_intern/modeling_long_vita.py:74-89 and :238-255, and the
composition of :90-221 (vision tower -> drop cls -> projector -> embedding gather + index_put ->
decoder layers -> final norm) and :309-311 (lm_head over the last `num_logits_to_keep` rows).
All arithmetic runs in liblvb200.so (long_vita_b200.ops); PyTorch holds the buffers.

`use_cache=True` returns a `kv_cache.KVCache` in `past_key_values` (pre-allocated, post-RoPE rows); a
later call with that cache and the new token(s) runs incremental decoding: one token -> the
flash-decoding composition `ops.attention_decode`, several tokens -> the fused kernel with the
bottom-right-aligned causal mask over cache + new rows (chunked prefill).  A cache that does not fit in HBM beside
the prefill (a ~1M-token prompt) is a `kv_cache.OffloadedKVCache` whose trailing layers live in pinned host memory
and are decoded in place (`ops.attention_decode_host`); see new_cache.  Images are encoded only when
the cache is empty (modeling_long_vita.py:90).  The Megatron serving path of the reference re-prefills
every token (long_vita_megatron/inference/text_generation/generation.py:127-135); SURVEY.md 8f-2.
"""
from __future__ import annotations

from dataclasses import dataclass
from functools import partial
from typing import Dict, Iterable, List, Optional, Tuple

import torch

from .. import kv_cache, ops
from ..config import LongVITAConfig
from ..kv_cache import ContextCache, ContextSession, KVCache, OffloadedKVCache


@dataclass
class CausalLMOutput:
    loss: Optional[torch.Tensor]
    logits: torch.Tensor
    past_key_values: Optional[object] = None
    hidden_states: Optional[Tuple[torch.Tensor, ...]] = None
    attentions: Optional[Tuple[torch.Tensor, ...]] = None

    def to_tuple(self):
        return tuple(v for v in (self.loss, self.logits, self.past_key_values, self.hidden_states) if v is not None)


@dataclass
class BaseOutput:
    last_hidden_state: torch.Tensor
    past_key_values: Optional[object] = None
    hidden_states: Optional[Tuple[torch.Tensor, ...]] = None
    attentions: Optional[Tuple[torch.Tensor, ...]] = None

    def to_tuple(self):
        return tuple(v for v in (self.last_hidden_state, self.past_key_values, self.hidden_states) if v is not None)

    def __getitem__(self, i):
        return self.to_tuple()[i]


class InternVisionModel:
    """InternViT-300M tower (modeling_intern_vit.py:298-363): patch-embed GEMM + cls + pos,
    24 x [LN -> MHA -> *ls1 + res -> LN -> fc1 -> GELU -> fc2 -> *ls2 + res]."""

    def __init__(self, cfg: LongVITAConfig, w: Dict[str, torch.Tensor], prefix: str = "model.vision_model."):
        self.cfg = cfg.visual
        v = self.cfg
        e = prefix + "embeddings."
        self.cls = w[e + "class_embedding"]
        self.pos = w[e + "position_embedding"]
        self.patch_w = ops.pad_patch_weight(w[e + "patch_embedding.weight"])
        self.patch_b = w[e + "patch_embedding.bias"]
        self.layers: List[Dict[str, torch.Tensor]] = []
        for i in range(v.num_hidden_layers):
            p = f"{prefix}encoder.layers.{i}."
            self.layers.append({k[len(p):]: t for k, t in w.items() if k.startswith(p)})

    def forward(self, pixel_values: torch.Tensor) -> torch.Tensor:
        v = self.cfg
        n = pixel_values.shape[0]
        C, H, D = v.hidden_size, v.num_attention_heads, v.head_dim
        x = ops.patch_embed(pixel_values, self.patch_w, self.patch_b, self.cls, self.pos, v.patch_size)
        S = x.shape[1]
        x = x.view(n * S, C)
        for L in self.layers:
            h = ops.layernorm(x, L["norm1.weight"], L["norm1.bias"], v.layer_norm_eps)
            qkv = ops.linear(h, L["attn.qkv.weight"], L.get("attn.qkv.bias")).view(n, S, 3, H, D)
            # 'b s (three h d)' (modeling_intern_vit.py:165): q/k/v are strided views, consumed in place
            att = ops.attention_fwd(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], causal=False, scale=D ** -0.5)
            o = ops.linear(att.view(n * S, C), L["attn.proj.weight"], L["attn.proj.bias"])
            x = ops.ls_residual(x, o, L["ls1"])
            h = ops.layernorm(x, L["norm2.weight"], L["norm2.bias"], v.layer_norm_eps)
            f = ops.linear(h, L["mlp.fc1.weight"], L["mlp.fc1.bias"], act="gelu")
            f = ops.linear(f, L["mlp.fc2.weight"], L["mlp.fc2.bias"])
            x = ops.ls_residual(x, f, L["ls2"])
        return x.view(n, S, C)

    __call__ = forward


class ResamplerProjector:
    """drop cls -> pixel-shuffle x0.5 -> LayerNorm(4C) -> Linear(4C, C) -> GELU -> Linear(C, hidden)
    (resampler_projector.py:26-34; the cls drop is modeling_long_vita.py:97, fused here)."""

    def __init__(self, cfg: LongVITAConfig, w: Dict[str, torch.Tensor], prefix: str = "model.vision_projection."):
        self.cfg = cfg
        self.ln_w = w[prefix + "pre_proj_layernorm.weight"]
        self.ln_b = w[prefix + "pre_proj_layernorm.bias"]
        self.w0 = w[prefix + "mlp.0.weight"]
        self.w2 = w[prefix + "mlp.2.weight"]

    def forward(self, vit_out: torch.Tensor, has_cls: bool = True) -> torch.Tensor:
        v = self.cfg.visual
        x = ops.pixel_shuffle(vit_out, v.grid, has_cls=has_cls)
        n, t, c4 = x.shape
        x = ops.layernorm(x.view(n * t, c4), self.ln_w, self.ln_b, v.pre_proj_ln_eps)
        x = ops.linear(x, self.w0, None, act="gelu")
        x = ops.linear(x, self.w2)
        return x.view(n, t, -1)

    __call__ = forward


# Row chunking of the decoder layer's token-wise work.  Up to ROW_CHUNK_THRESHOLD rows a layer runs each op once over
# all rows.  Above it, the ops before and after attention run on near-equal chunks of about ROW_CHUNK rows, so that
# only x, the QKV buffer, the attention output and the RoPE tables span the whole sequence: ~35 KB per token at the
# 14B geometry instead of ~103 KB (the whole-tensor layer also holds the [T, 13824] SwiGLU output, the MLP output and
# a second copy of x), which is what lets a ~1M-token prompt prefill on one 80 GB H100.
#
# Chunking is bit-identical to the whole-tensor call.  RMSNorm, RoPE and the residual add compute each row on its
# own, and their launch shape depends only on the column count.  The wgmma GEMM (gemm.cu) has no split-K: an output
# element is one accumulation over K in a fixed k-order, whatever M is, and since every chunk but the last starts
# at a multiple of its 128-row tile, each row even sits at the same place in its tile as in the whole call.  What
# would change the sum order is the GEMV path, which lv_gemm_bias_act takes for M <= 4, so no chunk is that short.
ROW_CHUNK_THRESHOLD = 262_144
ROW_CHUNK = 65_536
_ROW_ALIGN = 128            # the GEMM's M tile
_GEMV_MAX_ROWS = 4          # lv_gemm_bias_act's GEMV path


def row_chunks(T: int) -> List[Tuple[int, int]]:
    """The row spans [r0, r1) a decoder layer of T rows runs its token-wise ops on: [(0, T)] up to
    ROW_CHUNK_THRESHOLD rows, else near-equal chunks of about ROW_CHUNK rows, each a multiple of 128 rows but the
    last, and none of 4 rows or fewer."""
    if T <= ROW_CHUNK_THRESHOLD:
        return [(0, T)]
    n = -(-T // ROW_CHUNK)
    size = -(-T // (n * _ROW_ALIGN)) * _ROW_ALIGN
    spans = [(r, min(r + size, T)) for r in range(0, T, size)]
    if len(spans) > 1 and spans[-1][1] - spans[-1][0] <= _GEMV_MAX_ROWS:
        spans[-2:] = [(spans[-2][0], T)]
    return spans


# Streamed decoder layer.  Above STREAM_THRESHOLD rows, when the attention step is plain causal attention over this
# forward's rows, a layer runs everything, attention included, span by span in row order: rows [r0, r1) attend only
# to keys [0, r1), which are written by then.  Only x and one K|V buffer (shared by the layers of a forward) span the
# sequence: 14 848 B per token with the RoPE tables at the 14B geometry, against 35 328 for the row-chunked layer.
# The threshold lies between the 1M bench prompt (1 058 816 rows, row-chunked) and the ~1.33 M rows where the
# row-chunked layer runs out of memory on one 80 GB H100.
#
# Streaming is bit-identical to the whole call.  The QKV GEMM runs as two launches over row slices of the weight (Q
# columns, then K|V columns); with no split-K each output element keeps its k-order.  A query chunk over its key
# prefix is lv_attn_fwd with sq < sk, its mask aligned to the last key: its first row sits at global position r0, a
# multiple of 128, so every 128-row query item and every key tile is the one of the whole call.
STREAM_THRESHOLD = 1_179_648


def query_chunked(attend) -> bool:
    """Whether the attention step `attend` (bare or under functools.partial) declares `query_chunks`: it may be called
    with the query rows [r0, r1) over the keys [0, r1) and then returns exactly those rows of the whole call."""
    while isinstance(attend, partial):
        attend = attend.func
    return bool(getattr(attend, "query_chunks", False))


def streams(T: int, attend) -> bool:
    """Whether a decoder layer of T rows with the attention step `attend` runs streamed (STREAM_THRESHOLD)."""
    return T > STREAM_THRESHOLD and query_chunked(attend)


LINEAR_DTYPES = (torch.bfloat16, torch.float8_e4m3fn)
ATTN_DTYPES = (torch.bfloat16, torch.float8_e4m3fn)


def check_linear_dtype(linear_dtype) -> torch.dtype:
    """linear_dtype if it is a format of the decoder's linear weights (bf16, the default, or FP8 e4m3), else
    ValueError."""
    if linear_dtype not in LINEAR_DTYPES:
        raise ValueError(f"linear_dtype must be torch.bfloat16 or torch.float8_e4m3fn, got {linear_dtype!r}")
    return linear_dtype


def check_attn_dtype(attn_dtype) -> torch.dtype:
    """attn_dtype if it is an operand format of the decoder's prefill attention (bf16, the default, or FP8 e4m3:
    ops.attention_fwd_fp8), else ValueError."""
    if attn_dtype not in ATTN_DTYPES:
        raise ValueError(f"attn_dtype must be torch.bfloat16 or torch.float8_e4m3fn, got {attn_dtype!r}")
    return attn_dtype


class DecoderLayer:
    """Qwen2 decoder layer (transformers Qwen2DecoderLayer, instantiated by the reference at
    modeling_long_vita.py:57-72; mcore twin transformer_layer.py:173-257) with fused QKV and fused
    gate|up weights (layout of tools/hf2mcore_long_vita.py:486-504).

    With linear_dtype=torch.float8_e4m3fn the four linear weights are ops.Fp8Weight (e4m3, one scale per output
    channel), quantised here from the fused bf16 weights; ops.linear then runs the FP8 product at every call site.
    Biases and norm weights stay bf16."""

    def __init__(self, cfg: LongVITAConfig, w: Dict[str, torch.Tensor], i: int, linear_dtype=torch.bfloat16):
        p = f"model.layers.{i}."
        self.cfg = cfg
        self.wqkv = torch.cat([w[p + "self_attn.q_proj.weight"], w[p + "self_attn.k_proj.weight"],
                               w[p + "self_attn.v_proj.weight"]], dim=0).contiguous()
        self.bqkv = torch.cat([w[p + "self_attn.q_proj.bias"], w[p + "self_attn.k_proj.bias"],
                               w[p + "self_attn.v_proj.bias"]], dim=0).contiguous()
        self.wo = w[p + "self_attn.o_proj.weight"]
        # rows interleaved (gate_i, up_i): SwiGLU runs in the GEMM epilogue, [T, 2I] never touches HBM
        self.w_gate_up = ops.interleave_gate_up(w[p + "mlp.gate_proj.weight"], w[p + "mlp.up_proj.weight"])
        self.w_down = w[p + "mlp.down_proj.weight"]
        self.ln1 = w[p + "input_layernorm.weight"]
        self.ln2 = w[p + "post_attention_layernorm.weight"]
        if check_linear_dtype(linear_dtype) == torch.float8_e4m3fn:
            for name in ("wqkv", "wo", "w_gate_up", "w_down"):
                setattr(self, name, ops.Fp8Weight.quantize(getattr(self, name)))

    def linear_bytes(self) -> int:
        """Resident bytes of the four linear weights (with their scales in FP8)."""
        return sum(t.nbytes() if isinstance(t, ops.Fp8Weight) else t.numel() * t.element_size()
                   for t in (self.wqkv, self.wo, self.w_gate_up, self.w_down))

    def forward(self, x: torch.Tensor, delta: Optional[torch.Tensor], cos, sin, attend,
                qkv_out: Optional[torch.Tensor] = None,
                inplace: bool = False,
                kv_out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """x [T, H] residual stream, `delta` the previous layer's MLP output not yet added (the add is fused into this
        layer's first RMSNorm), or None.  Returns (x, delta).

        `attend(q, k, v)` is the attention step: q [T, hq, d], k / v [T, hkv, d] are views of the QKV GEMM output,
        after RoPE (skipped when `cos` is None); it returns the attention output ([T, hq * d] in any shape).
        `qkv_out` is a caller buffer [T, (hq + 2 hkv) d] for the QKV GEMM, e.g. the peer-mapped buffer that the
        context-parallel kernel reads the other ranks' K/V from.

        Above ROW_CHUNK_THRESHOLD rows the ops before and after attention run chunk by chunk (row_chunks); attention
        is still one call over all rows, enqueued after every QKV row is written.  Each chunk's MLP output is then
        added to its rows of x at once and the returned delta is None.  With several chunks and `inplace`, x itself
        is that residual stream (its rows are overwritten); otherwise the layer writes a new one.

        Above STREAM_THRESHOLD rows, with an attention step that declares `query_chunks` (query_chunked), the layer
        streams: every op, attention included, runs span by span, each span's queries over the keys up to its last
        row.  K|V rows go to `kv_out` [T, 2 hkv d] (allocated here if None), and x and delta as above."""
        cfg = self.cfg
        T = x.shape[0]
        spans = row_chunks(T)
        if streams(T, attend):
            if qkv_out is not None:
                raise ValueError("DecoderLayer.forward: a streamed layer writes Q per span and K|V to kv_out; it takes "
                                 "no qkv_out")
            return self._forward_streamed(x, delta, cos, sin, attend, kv_out, spans, inplace)
        if len(spans) > 1:
            return self._forward_chunked(x, delta, cos, sin, attend, qkv_out, spans, inplace)
        hq, hkv, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        if delta is None:
            h = ops.rmsnorm(x, self.ln1, cfg.rms_norm_eps)
        else:
            h, x = ops.rmsnorm(delta, self.ln1, cfg.rms_norm_eps, residual=x)
        qkv = ops.linear(h, self.wqkv, self.bqkv, out=qkv_out)            # [T, (hq + 2 hkv) d]
        q = qkv[:, : hq * d].view(T, hq, d)
        k = qkv[:, hq * d : (hq + hkv) * d].view(T, hkv, d)
        v = qkv[:, (hq + hkv) * d :].view(T, hkv, d)
        if cos is not None:
            ops.rope(q, cos, sin, out=q)
            ops.rope(k, cos, sin, out=k)
        o = ops.linear(attend(q, k, v).reshape(T, hq * d), self.wo)
        h, x = ops.rmsnorm(o, self.ln2, cfg.rms_norm_eps, residual=x)
        a = ops.linear(h, self.w_gate_up, act="swiglu")
        return x, ops.linear(a, self.w_down)

    def _forward_chunked(self, x, delta, cos, sin, attend, qkv_out, spans, inplace):
        """forward() over the row spans `spans`: the same ops, each on its rows of x, the QKV buffer and the RoPE
        tables; returns (x with this layer's MLP output added, None)."""
        cfg = self.cfg
        T = x.shape[0]
        hq, hkv, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        eps = cfg.rms_norm_eps
        qkv = qkv_out if qkv_out is not None else torch.empty((T, (hq + 2 * hkv) * d), dtype=x.dtype, device=x.device)
        q = qkv[:, : hq * d].view(T, hq, d)
        k = qkv[:, hq * d : (hq + hkv) * d].view(T, hkv, d)
        v = qkv[:, (hq + hkv) * d :].view(T, hkv, d)
        xs = x if delta is None or inplace else torch.empty_like(x)         # x + delta
        for r0, r1 in spans:
            if delta is None:
                h = ops.rmsnorm(x[r0:r1], self.ln1, eps)
            else:
                h, _ = ops.rmsnorm(delta[r0:r1], self.ln1, eps, residual=x[r0:r1], out=xs[r0:r1])
            ops.linear(h, self.wqkv, self.bqkv, out=qkv[r0:r1])
            if cos is not None:
                ops.rope(q[r0:r1], cos[r0:r1], sin[r0:r1], out=q[r0:r1])
                ops.rope(k[r0:r1], cos[r0:r1], sin[r0:r1], out=k[r0:r1])
        x, h, delta = xs, None, None
        o = attend(q, k, v).reshape(T, hq * d)
        del q, k, v, qkv                    # the QKV buffer is released (unless it is the caller's) before the MLP
        xo = x if inplace else torch.empty_like(x)
        for r0, r1 in spans:
            h, _ = ops.rmsnorm(ops.linear(o[r0:r1], self.wo), self.ln2, eps, residual=x[r0:r1], out=xo[r0:r1])
            m = ops.linear(ops.linear(h, self.w_gate_up, act="swiglu"), self.w_down)
            ops.ls_residual(xo[r0:r1], m, out=xo[r0:r1])      # the add the next layer's first RMSNorm would fuse
        return xo, None

    def _forward_streamed(self, x, delta, cos, sin, attend, kv, spans, inplace):
        """forward() with every op on the row spans `spans` in order (STREAM_THRESHOLD): Q of a span in a span buffer,
        its K|V rows into `kv`, attention of the span's queries over kv[:r1]; returns (x with this layer's MLP output
        added, None).  A span reads no row of x but its own, so x may be the residual stream it writes."""
        cfg = self.cfg
        T = x.shape[0]
        hq, hkv, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        eps = cfg.rms_norm_eps
        nq = hq * d
        if kv is None:
            kv = torch.empty((T, 2 * hkv * d), dtype=x.dtype, device=x.device)
        k = kv[:, : hkv * d].view(T, hkv, d)
        v = kv[:, hkv * d :].view(T, hkv, d)
        xo = x if inplace else torch.empty_like(x)
        for r0, r1 in spans:
            n = r1 - r0
            if delta is None:
                h, res = ops.rmsnorm(x[r0:r1], self.ln1, eps), x[r0:r1]
            else:
                h, res = ops.rmsnorm(delta[r0:r1], self.ln1, eps, residual=x[r0:r1], out=xo[r0:r1])
            q = ops.linear(h, self.wqkv[:nq], self.bqkv[:nq]).view(n, hq, d)
            ops.linear(h, self.wqkv[nq:], self.bqkv[nq:], out=kv[r0:r1])
            if cos is not None:
                ops.rope(q, cos[r0:r1], sin[r0:r1], out=q)
                ops.rope(k[r0:r1], cos[r0:r1], sin[r0:r1], out=k[r0:r1])
            o = attend(q, k[:r1], v[:r1]).reshape(n, nq)
            h, _ = ops.rmsnorm(ops.linear(o, self.wo), self.ln2, eps, residual=res, out=xo[r0:r1])
            m = ops.linear(ops.linear(h, self.w_gate_up, act="swiglu"), self.w_down)
            ops.ls_residual(xo[r0:r1], m, out=xo[r0:r1])
        return xo, None


def run_layers(layers, x: torch.Tensor, cos, sin, attend, norm_w: torch.Tensor, eps: float, *, cache=None,
               qkv_out=None, hidden: Optional[list] = None, donate: bool = False) -> torch.Tensor:
    """The decoder stack: x [T, H] embeddings -> the final RMSNorm of the last hidden state [T, H].

    Each layer's MLP output is handed on as `delta` and added inside the next RMSNorm (the last one inside the final
    norm); a layer that runs in row chunks (row_chunks) adds it itself.  `attend(layer_index, q, k, v)` is the
    attention step (DecoderLayer.forward); `qkv_out()`, if given, the QKV GEMM's output buffer of the next layer.  The
    K/V rows appended to `cache` during the pass are committed at its end.  `hidden` (a list) receives each layer's
    input hidden state.  `donate`: x was made for this call (an embedding output), so chunked layers may update it in
    place; the stack's own residual stream is updated in place from the second layer on (unless `hidden` keeps it).
    Streamed layers (STREAM_THRESHOLD) share one K|V buffer, allocated here."""
    delta = None
    kv = None
    if layers and streams(x.shape[0], attend):
        c = layers[0].cfg
        kv = torch.empty((x.shape[0], 2 * c.num_key_value_heads * c.head_dim), dtype=x.dtype, device=x.device)
    for li, layer in enumerate(layers):
        if hidden is not None:
            hidden.append(x if delta is None else x + delta)
        x, delta = layer.forward(x, delta, cos, sin, partial(attend, li), None if qkv_out is None else qkv_out(),
                                 inplace=(donate or li > 0) and hidden is None, kv_out=kv)
    if cache is not None:
        cache.commit()
    if kv is not None:
        # streamed: x is the stack's own residual stream (the layers replaced or donated it); the final norm writes it
        # span by span, so that no second [T, H] tensor exists beside it
        del kv
        for r0, r1 in row_chunks(x.shape[0]):
            x[r0:r1].copy_(ops.rmsnorm(x[r0:r1], norm_w, eps))
        return x
    if delta is None:
        return ops.rmsnorm(x, norm_w, eps)
    return ops.rmsnorm(delta, norm_w, eps, residual=x)[0]


def prefill_bytes_per_token(cfg: LongVITAConfig, T: int, streamed: bool, linear_dtype=torch.bfloat16,
                            attn_dtype=torch.bfloat16) -> int:
    """Device bytes per token that a decoder prefill of T rows holds beside the weights (DESIGN §3): whole-tensor
    layer (x, delta, QKV, attention output, new x, norm output, SwiGLU output, MLP output), row-chunked layer (x, QKV,
    attention output) or streamed layer (x, K|V), plus the RoPE tables.  At the 14B geometry: 103 936, 35 328 and
    14 848 B.  With FP8 linears, add the largest quantised A operand (e4m3 rows of the widest linear input and their
    fp32 scales) over the longest row span, spread over the T rows.  With FP8 attention, add the quantised K / V of a
    call over all T keys (ops.attn_fp8_kv_bytes: 2 hkv d bytes per key row and the block scales)."""
    H, I = cfg.hidden_size, cfg.intermediate_size
    hq, hkv, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    rope = 2 * 2 * d
    fp8 = 0
    if linear_dtype == torch.float8_e4m3fn and T > 0:
        span = max(r1 - r0 for r0, r1 in row_chunks(T))
        fp8 = -(-span * (max(H, hq * d, I) + 4) // T)
    if attn_dtype == torch.float8_e4m3fn and T > 0:
        fp8 += -(-ops.attn_fp8_kv_bytes(T, hkv, d) // T)
    if streamed:
        return 2 * (H + 2 * hkv * d) + rope + fp8
    if len(row_chunks(T)) > 1:
        return 2 * (H + (hq + 2 * hkv) * d + hq * d) + rope + fp8
    return 2 * (5 * H + hq * d + (hq + 2 * hkv) * d + I) + rope + fp8


def new_cache(cfg: LongVITAConfig, num_layers: int, capacity: int, rows: int, device,
              host_dtype=torch.bfloat16, linear_dtype=torch.bfloat16, attn_dtype=torch.bfloat16):
    """The K/V cache of a generation whose prompt has `rows` tokens (kv_cache.make_cache): on the device when it fits
    beside that prompt's prefill (with `linear_dtype` linears and `attn_dtype` attention), else partly in pinned host
    memory (in `host_dtype`: bf16, or the lossy FP8 e4m3 format), in which case the prefill streams above
    STREAM_THRESHOLD (attention_step)."""
    return kv_cache.make_cache(num_layers, capacity, cfg.num_key_value_heads, cfg.head_dim, device,
                               prefill_bytes=rows * prefill_bytes_per_token(cfg, rows, False, linear_dtype, attn_dtype),
                               offloaded_prefill_bytes=rows * prefill_bytes_per_token(cfg, rows,
                                                                                      rows > STREAM_THRESHOLD,
                                                                                      linear_dtype, attn_dtype),
                               host_dtype=host_dtype)


def attention_step(cache=None, cu_seqlens: Optional[torch.Tensor] = None, rows: int = 1, attn_dtype=torch.bfloat16):
    """The single-GPU attention step for run_layers.  Without `cache`: causal attention over this forward's rows
    (inside each packed document with `cu_seqlens`).  With `cache`: the new K/V rows are appended to it and one new
    token attends over the whole cache (flash-decoding), several new tokens over cache + new rows with the causal mask
    aligned to the last key (the first prefill, or a chunk).

    With a kv_cache.OffloadedKVCache, a layer on the host tier copies its new rows to its host buffer; in the prefill
    it then attends over its own k, v exactly as the step without a cache does, and a new token attends over the
    host rows in place (ops.attention_decode_host, or ops.attention_decode_host_fp8 for an FP8 host tier; the prefill
    never reads the host rows, so its logits do not depend on the host format).  `rows` is the number of new tokens
    of the forward; a cache that cannot take them raises before anything is launched.

    The plain step (no cache, one sample) and the prefill step of an empty offloaded cache declare `query_chunks`
    (query_chunked): called with query rows [r0, r1) and the keys [0, r1), its mask aligned to the last key gives
    exactly those rows of the whole call.

    `attn_dtype=torch.float8_e4m3fn` runs every call of several new tokens on the FP8 kernel (ops.attention_fwd_fp8:
    lossy, opt-in), whole-tensor, row-chunked and streamed alike; its blocks are aligned to key row 0, so the span
    calls of the streamed layer still give exactly the rows of the whole call.  One new token (decode) and the cache
    contents stay bf16.  Packed rows (`cu_seqlens`) have no FP8 path: NotImplementedError, before anything runs.

    With a kv_cache.ContextSession (a question about a prefilled context) see context_step."""
    fp8 = check_attn_dtype(attn_dtype) == torch.float8_e4m3fn
    if fp8 and cu_seqlens is not None:
        raise NotImplementedError("packed samples (position ids restarting at 0) have no FP8 attention; use "
                                  "attn_dtype=torch.bfloat16")
    docs = ops.docs_kwargs(cu_seqlens)
    if isinstance(cache, ContextSession):
        if cu_seqlens is not None:
            raise NotImplementedError(PACKED_WITH_CACHE)
        return context_step(cache, rows)

    def prefill(q, k, v, **kw):
        fwd = ops.attention_fwd_fp8 if fp8 else ops.attention_fwd
        return fwd(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0), causal=True, **kw)

    if cache is None:
        def attend(li, q, k, v):
            return prefill(q, k, v, **docs)

        attend.query_chunks = cu_seqlens is None
        return attend

    if isinstance(cache, OffloadedKVCache):
        cache.check_rows(rows)

        def attend(li, q, k, v):
            n = q.shape[0]
            if cache.on_host(li):
                kh, length = cache.append_host(li, k, v, n)
                if n == 1:
                    return cache.decode_host(q[0], kh, length)
                return prefill(q, k, v)
            kc, vc, length = cache.append(li, k, v, n)
            if n == 1:
                return ops.attention_decode(q[0], kc, vc, length)
            return prefill(q, kc[:length], vc[:length])

        attend.query_chunks = len(cache) == 0
        return attend

    def attend(li, q, k, v):
        kc, vc, length = cache.append(li, k, v)
        if q.shape[0] == 1:
            return ops.attention_decode(q[0], kc, vc, length)
        return prefill(q, kc[:length], vc[:length])

    return attend


def context_step(session: ContextSession, rows: int):
    """The attention step of a question about a prefilled context: each layer appends its new K/V rows to the session's
    suffix, then attends its new rows over the context's P rows and over the suffix, each part with its log-sum-exp,
    and merges the two parts (ops.merge_attention).

    The context part is unmasked: on a device layer ops.attention_fwd over K[:P] (ops.attention_decode for one row),
    on a host layer ops.attention_host_rows (ops.attention_decode_host or _fp8 for one row).  The suffix part is causal
    attention over the suffix rows, aligned to the last key (ops.attention_decode for one row).  A question runs bf16
    attention whatever the model's attn_dtype, as decode steps do.  A question that overflows the suffix raises before
    anything is launched."""
    session.check_rows(rows)
    ctx, P = session.context.cache, session.prefix_len

    def attend(li, q, k, v):
        n, hq, d = q.shape
        kc, vc, length = session.suffix.append(li, k, v)
        if isinstance(ctx, OffloadedKVCache) and ctx.on_host(li):
            host = ctx.host[li - ctx.n_dev]
            if n == 1:
                o1, l1 = ctx.decode_host(q[0], host, P, return_lse=True)
            else:
                o1, l1 = ops.attention_host_rows(q, host, P, return_lse=True)
        elif n == 1:
            o1, l1 = ops.attention_decode(q[0], ctx.k[li], ctx.v[li], P, return_lse=True)
        else:
            o1, l1 = ops.attention_fwd(q.unsqueeze(0), ctx.k[li][:P].unsqueeze(0), ctx.v[li][:P].unsqueeze(0),
                                       causal=False, return_lse=True)
        if n == 1:
            o2, l2 = ops.attention_decode(q[0], kc, vc, length, return_lse=True)
        else:
            o2, l2 = ops.attention_fwd(q.unsqueeze(0), kc[:length].unsqueeze(0), vc[:length].unsqueeze(0), causal=True,
                                       return_lse=True)
        return ops.merge_attention(torch.stack([o1.view(n, hq, d), o2.view(n, hq, d)]),
                                   torch.stack([l1.view(hq, n), l2.view(hq, n)]))

    return attend


PACKED_WITH_CACHE = ("packed samples (position ids restarting at 0) cannot be combined with a KV cache "
                     "(use_cache / past_key_values / inference_params)")


def packed_rows(position_ids: torch.Tensor, seq_len: int, device, *, cache=None, cp=None) -> Optional[torch.Tensor]:
    """cu_seqlens of a packed row (position ids restarting at 0 mark the sample boundaries; one host synchronisation),
    or None when the row holds one sample.  Packing under context parallelism (`cp`) or with a K/V cache raises."""
    cu = ops.packed_cu_seqlens(position_ids, device=device, seq_len=seq_len)
    if cu is not None:
        if cp is not None:
            raise NotImplementedError("packed samples (position ids restarting at 0) under context parallelism are "
                                      "not supported")
        if cache is not None:
            raise NotImplementedError(PACKED_WITH_CACHE)
    return cu


def rope_inv_freq(cfg: LongVITAConfig, device) -> torch.Tensor:
    """Qwen2's RoPE frequencies 1 / theta^(2i / d), fp32."""
    return (1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2, dtype=torch.int64).float()
                                      / cfg.head_dim))).to(device)


VISION_CHUNK = 256  # frames per ViT pass (MegatronVisionModel.forward_chunk, pretrain_long_vita.py:522-533)


def vision_tower(cfg: LongVITAConfig, w: Dict[str, torch.Tensor]):
    """(InternVisionModel, ResamplerProjector), or (None, None) for weights without a vision tower."""
    if "model.vision_model.embeddings.class_embedding" not in w:
        return None, None
    return InternVisionModel(cfg, w), ResamplerProjector(cfg, w)


def encode_images(vision_model, projection, images: torch.Tensor, chunk: int = VISION_CHUNK) -> torch.Tensor:
    """images [n, 3, 448, 448] -> projected features [n, tokens_per_image, H], `chunk` frames per ViT pass."""
    feats = []
    for i in range(0, images.shape[0], chunk):
        feats.append(projection(vision_model(images[i : i + chunk]), has_cls=True))
    return feats[0] if len(feats) == 1 else torch.cat(feats, dim=0)


def scatter_images(x: torch.Tensor, vision_model, projection, images: torch.Tensor, dst: torch.Tensor,
                   chunk: int = VISION_CHUNK) -> torch.Tensor:
    """Writes the projected features of `images` into the rows `dst` of the embedded prompt x [T, H] (image-major:
    each image's tokens_per_image rows in turn) and returns x.  Each `chunk` frames' features are scattered as soon
    as they are made, so the whole-prompt feature tensor of encode_images never exists (21.5 GB at 8192 frames).
    For unique `dst` the result is bit-identical to ops.embed_scatter with encode_images' features."""
    n = images.shape[0]
    if n == 0 or dst.numel() % n:
        raise ValueError(f"scatter_images: {dst.numel()} target rows for {n} images")
    tpi = dst.numel() // n
    for i in range(0, n, chunk):
        feat = projection(vision_model(images[i : i + chunk]), has_cls=True)
        ops.row_scatter(feat, dst[i * tpi : (i + feat.shape[0]) * tpi], x)
    return x


def _map_tensors(obj, fn, seen=None):
    """Apply `fn` to every tensor reachable from the attributes of our plain weight holders (in place)."""
    seen = set() if seen is None else seen
    if id(obj) in seen:
        return
    seen.add(id(obj))
    items = obj.items() if isinstance(obj, dict) else vars(obj).items()
    for name, val in list(items):
        if isinstance(val, torch.Tensor):
            new = fn(val)
            if isinstance(obj, dict):
                obj[name] = new
            else:
                object.__setattr__(obj, name, new)
        elif isinstance(val, (list, tuple)):
            for i, e in enumerate(val):
                if isinstance(e, torch.Tensor):
                    val[i] = fn(e)
                elif isinstance(e, (dict, InternVisionModel, ResamplerProjector, DecoderLayer)):
                    _map_tensors(e, fn, seen)
        elif isinstance(val, (dict, InternVisionModel, ResamplerProjector, DecoderLayer)):
            _map_tensors(val, fn, seen)
        elif isinstance(val, ops.Fp8Weight):
            # moved, never cast: fn applied to the fp32 scale says where the weight goes
            new = val.to(fn(val.scale).device)
            if isinstance(obj, dict):
                obj[name] = new
            else:
                object.__setattr__(obj, name, new)


class _WeightHolderModule(torch.nn.Module):
    """nn.Module whose weights live in plain tensors (fused / re-laid-out once at load for the kernels) rather than in
    nn.Parameters: `.to()` / `.cuda()` / `.eval()` / hooks work as for any module, `state_dict()` is rebuilt in the
    reference's HF names by the subclasses."""

    def _apply(self, fn, recurse=True):
        super()._apply(fn, recurse)
        _map_tensors(self, lambda t: fn(t) if t.is_floating_point() or t.dtype in (torch.int64, torch.int32) else t)
        return self


class LongVITAModel(_WeightHolderModule):
    def __init__(self, cfg: LongVITAConfig, weights: Dict[str, torch.Tensor],
                 layers: Optional[Iterable[DecoderLayer]] = None, linear_dtype=torch.bfloat16,
                 attn_dtype=torch.bfloat16):
        """`layers` replaces the decoder layers of `weights` (e.g. layers built one at a time, so that a layer's
        unfused q/k/v and gate/up weights are freed before the next one is drawn); they must have been built with
        `linear_dtype`, the format of the decoder's linear weights (bf16, or FP8 e4m3: DecoderLayer).  `attn_dtype`
        is the operand format of the decoder's prefill attention (bf16, or FP8 e4m3: attention_step)."""
        super().__init__()
        self.config = cfg
        self.linear_dtype = check_linear_dtype(linear_dtype)
        self.attn_dtype = check_attn_dtype(attn_dtype)
        self.embed_tokens = weights["model.embed_tokens.weight"]
        self.norm_w = weights["model.norm.weight"]
        self.layers = ([DecoderLayer(cfg, weights, i, linear_dtype) for i in range(cfg.num_hidden_layers)]
                       if layers is None else list(layers))
        fp8 = linear_dtype == torch.float8_e4m3fn
        for i, layer in enumerate(self.layers):
            if isinstance(layer.wqkv, ops.Fp8Weight) != fp8:
                raise ValueError(f"decoder layer {i} was not built with linear_dtype={linear_dtype}")
        self.vision_model, self.vision_projection = vision_tower(cfg, weights)
        self.inv_freq = rope_inv_freq(cfg, self.embed_tokens.device)
        self.vision_chunk = VISION_CHUNK
        self.default_new_tokens = 1024   # head-room of a cache created by use_cache=True (max_cache_len= overrides)

    def encode_images(self, images: torch.Tensor) -> torch.Tensor:
        return encode_images(self.vision_model, self.vision_projection, images, self.vision_chunk)

    def forward(
        self,
        input_ids: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        images: Optional[torch.Tensor] = None,
        image_indices: Optional[torch.Tensor] = None,
        position_ids: Optional[torch.Tensor] = None,
        past_key_values=None,
        inputs_embeds: Optional[torch.Tensor] = None,
        use_cache: Optional[bool] = None,
        output_attentions: Optional[bool] = None,
        output_hidden_states: Optional[bool] = None,
        return_dict: Optional[bool] = None,
        cache_position: Optional[torch.Tensor] = None,
        **flash_attn_kwargs,
    ):
        cfg = self.config
        if (input_ids is None) ^ (inputs_embeds is not None):
            raise ValueError("You must specify exactly one of input_ids or inputs_embeds")
        if isinstance(past_key_values, ContextCache):
            raise TypeError("a ContextCache is read-only: pass past_key_values=context.session(max_new_rows), a "
                            "session with room for the question's and the answer's rows")
        if past_key_values is not None and not isinstance(past_key_values, (KVCache, OffloadedKVCache,
                                                                            ContextSession)):
            if len(past_key_values) != 0:
                raise NotImplementedError("past_key_values must be the KVCache returned by a use_cache=True call")
            past_key_values = None
        if output_attentions:
            raise NotImplementedError("attention probabilities are never materialised by the fused kernel")
        if attention_mask is not None and not bool(attention_mask.to(torch.bool).all()):
            raise NotImplementedError("padding masks are not supported; pass unpadded sequences (batch 1)")

        past_len = 0 if past_key_values is None else past_key_values.get_seq_length()
        if inputs_embeds is None:
            b, s = input_ids.shape
            if b != 1:
                raise NotImplementedError("batch size 1 (the reference's long-context configuration)")
            dev = self.embed_tokens.device
        else:
            b, s, _ = inputs_embeds.shape
            if b != 1:
                raise NotImplementedError("batch size 1")
            dev = inputs_embeds.device

        cache = past_key_values
        # kv_host_dtype: the format of the host tier of a cache this call creates (kv_cache.make_cache)
        host_dtype = kv_cache.check_host_dtype(flash_attn_kwargs.pop("kv_host_dtype", torch.bfloat16))
        if use_cache and cache is None:
            capacity = int(flash_attn_kwargs.pop("max_cache_len", 0)) or s + self.default_new_tokens
            cache = new_cache(cfg, len(self.layers), capacity, s, dev, host_dtype, self.linear_dtype, self.attn_dtype)
        flash_attn_kwargs.pop("max_cache_len", None)
        if cache_position is None:
            cache_position = torch.arange(past_len, past_len + s, device=dev)     # modeling_long_vita.py:153-158
        cu = None
        if position_ids is None:
            position_ids = cache_position.unsqueeze(0)
        else:
            # packed samples: positions restarting at 0 inside the row are sample boundaries; attention stays inside
            # each sample, as transformers' flash_attention_2 does for the reference (tools/inference_long_vita.py:816)
            cu = packed_rows(position_ids, s, dev, cache=cache)
        attend = attention_step(cache, cu, s, self.attn_dtype)

        encode = images is not None and past_len == 0              # modeling_long_vita.py:90
        # when the decoder streams, so does the vision phase: each ViT chunk's features go into x as they are made
        stream_images = encode and inputs_embeds is None and streams(s, attend)
        image_embeds = None
        if encode and not stream_images:
            image_embeds = self.encode_images(images)
            assert image_embeds.shape[0] == len(images)

        if inputs_embeds is None:
            if encode:
                idx_b, idx_s = image_indices.to(input_ids.device).unbind(dim=0)
                dst = (idx_b.reshape(-1) * s + idx_s.reshape(-1)).to(torch.int64)
                if stream_images:
                    x = scatter_images(ops.embed_scatter(input_ids, self.embed_tokens), self.vision_model,
                                       self.vision_projection, images, dst, self.vision_chunk)
                else:
                    x = ops.embed_scatter(input_ids, self.embed_tokens, image_embeds, dst)
                image_embeds = None                 # scattered into x: not held through the decoder
            else:
                x = ops.embed_scatter(input_ids, self.embed_tokens)
        else:
            x = inputs_embeds.reshape(s, -1).contiguous()
        cos, sin = ops.rope_table(position_ids.reshape(-1).to(torch.int64), self.inv_freq)

        hidden = [] if output_hidden_states else None
        h = run_layers(self.layers, x, cos, sin, attend, self.norm_w, cfg.rms_norm_eps, cache=cache,
                       hidden=hidden, donate=inputs_embeds is None).view(1, s, -1)
        all_hidden = tuple(t.view(1, s, -1) for t in hidden) + (h,) if output_hidden_states else None
        out = BaseOutput(last_hidden_state=h, past_key_values=cache, hidden_states=all_hidden)
        return out if (return_dict is None or return_dict) else out.to_tuple()

    def hf_state_dict(self, prefix: str = "model.") -> Dict[str, torch.Tensor]:
        """The weights under the reference's HF parameter names (views of the fused buffers; the padded patch-embed
        operand is cut back to the [C, 3, ps, ps] conv weight).  A model with FP8 linears has no such state dict (no
        quantised checkpoint format is defined): NotImplementedError."""
        if self.linear_dtype != torch.bfloat16:
            raise NotImplementedError("state_dict() of a model with FP8 linears: no quantised checkpoint format is "
                                      "defined; load the bf16 checkpoint with linear_dtype= instead")
        sd = {prefix + "embed_tokens.weight": self.embed_tokens, prefix + "norm.weight": self.norm_w}
        cfg = self.config
        for i, L in enumerate(self.layers):
            p = f"{prefix}layers.{i}."
            q, kv = cfg.q_size, cfg.kv_size
            sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.q_proj.bias"] = L.wqkv[:q], L.bqkv[:q]
            sd[p + "self_attn.k_proj.weight"], sd[p + "self_attn.k_proj.bias"] = L.wqkv[q : q + kv], L.bqkv[q : q + kv]
            sd[p + "self_attn.v_proj.weight"], sd[p + "self_attn.v_proj.bias"] = L.wqkv[q + kv :], L.bqkv[q + kv :]
            sd[p + "self_attn.o_proj.weight"] = L.wo
            sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"] = L.w_gate_up[0::2], L.w_gate_up[1::2]
            sd[p + "mlp.down_proj.weight"] = L.w_down
            sd[p + "input_layernorm.weight"], sd[p + "post_attention_layernorm.weight"] = L.ln1, L.ln2
        if self.vision_model is not None:
            v, vm = cfg.visual, self.vision_model
            e = prefix + "vision_model.embeddings."
            sd[e + "class_embedding"], sd[e + "position_embedding"] = vm.cls, vm.pos
            k = 3 * v.patch_size * v.patch_size
            sd[e + "patch_embedding.weight"] = vm.patch_w[:, :k].reshape(-1, 3, v.patch_size, v.patch_size)
            sd[e + "patch_embedding.bias"] = vm.patch_b
            for i, L in enumerate(vm.layers):
                for name, t in L.items():
                    sd[f"{prefix}vision_model.encoder.layers.{i}.{name}"] = t
            pj = self.vision_projection
            q = prefix + "vision_projection."
            sd[q + "pre_proj_layernorm.weight"], sd[q + "pre_proj_layernorm.bias"] = pj.ln_w, pj.ln_b
            sd[q + "mlp.0.weight"], sd[q + "mlp.2.weight"] = pj.w0, pj.w2
        return sd


class GenerationDefaults:
    """The fields of transformers' GenerationConfig this build reads; `model.generation_config` may be replaced by a
    real GenerationConfig (tools/inference_long_vita.py:819-826 assigns one and then sets these attributes)."""

    def __init__(self):
        self.max_new_tokens = 1024
        self.do_sample = False
        self.use_cache = True
        self.eos_token_id = None
        self.pad_token_id = None


class LongVITAForCausalLM(_WeightHolderModule):
    def __init__(self, cfg: LongVITAConfig, weights: Dict[str, torch.Tensor],
                 layers: Optional[Iterable[DecoderLayer]] = None, linear_dtype=torch.bfloat16,
                 attn_dtype=torch.bfloat16):
        """`linear_dtype=torch.float8_e4m3fn` runs the decoder's four linears in FP8 (lossy, opt-in; DecoderLayer):
        their weights are quantised per output channel as the layers are built.  `attn_dtype=torch.float8_e4m3fn` runs
        the decoder's prefill attention on the FP8 kernel (lossy, opt-in; attention_step).  The vision tower,
        projector, embedding, norms and LM head stay bf16."""
        super().__init__()
        self.config = cfg
        self.model = LongVITAModel(cfg, weights, layers, linear_dtype, attn_dtype)
        self.lm_head = weights["lm_head.weight"]
        self.generation_config = GenerationDefaults()

    @property
    def device(self) -> torch.device:
        return self.lm_head.device

    @property
    def dtype(self) -> torch.dtype:
        return self.lm_head.dtype

    def state_dict(self, *args, **kwargs) -> Dict[str, torch.Tensor]:
        sd = self.model.hf_state_dict("model.")
        sd["lm_head.weight"] = self.lm_head
        return sd

    @classmethod
    def from_pretrained(cls, model_path: str, torch_dtype=torch.bfloat16, device_map=None, attn_implementation=None,
                        trust_remote_code: bool = True, linear_dtype=torch.bfloat16, attn_dtype=torch.bfloat16,
                        **kwargs):
        """Load a Long-VITA HF checkpoint directory (config.json + *.safetensors shards), the call
        tools/inference_long_vita.py:811-817 makes through AutoModelForCausalLM.  Only bfloat16 runs on the fused
        path; `attn_implementation` is accepted and ignored (the fused kernel IS the attention implementation);
        `device_map` "auto" / None -> the current CUDA device.  Decoder layers are read and built one at a time;
        `linear_dtype=torch.float8_e4m3fn` quantises each one's linears as it is built, `attn_dtype` selects the
        prefill attention (see __init__)."""
        import glob
        import json
        import os

        from safetensors import safe_open

        if torch_dtype not in (torch.bfloat16, "bfloat16", None, "auto"):
            raise NotImplementedError("the fused path computes in bfloat16 (the reference's torch_dtype)")
        check_linear_dtype(linear_dtype)
        check_attn_dtype(attn_dtype)
        c = json.load(open(os.path.join(model_path, "config.json")))
        vc = c.get("visual", c.get("vision_config", {})) or {}
        from dataclasses import fields, replace

        from ..config import VisionConfig

        def pick(dc, src):
            names = {f.name for f in fields(dc)}
            return {k: v for k, v in src.items() if k in names and not isinstance(v, dict)}

        cfg = replace(LongVITAConfig(**pick(LongVITAConfig, c)), visual=VisionConfig(**pick(VisionConfig, vc)))
        dev = torch.device("cuda", torch.cuda.current_device()) if device_map in (None, "auto") else torch.device(device_map)
        shards = sorted(glob.glob(os.path.join(model_path, "*.safetensors")))
        if not shards:
            raise FileNotFoundError(f"no *.safetensors under {model_path}")
        where: Dict[str, str] = {}
        for sh in shards:
            with safe_open(sh, framework="pt", device=str(dev)) as f:
                where.update((name, sh) for name in f.keys())

        def read(names):
            out: Dict[str, torch.Tensor] = {}
            for sh in sorted({where[n] for n in names}):
                with safe_open(sh, framework="pt", device=str(dev)) as f:
                    out.update((n, f.get_tensor(n).to(torch.bfloat16)) for n in names if where[n] == sh)
            return out

        # the decoder layers one at a time: a layer's bf16 tensors are released once it is built
        def layer_names(i):
            return [n for n in where if n.startswith(f"model.layers.{i}.")]

        w = read([n for n in where if not n.startswith("model.layers.")])
        layers = (DecoderLayer(cfg, read(layer_names(i)), i, linear_dtype) for i in range(cfg.num_hidden_layers))
        return cls(cfg, w, layers, linear_dtype, attn_dtype)

    @classmethod
    def from_synthetic(cls, cfg: LongVITAConfig, seed: int = 1234, device="cuda", perturb: bool = False,
                       num_layers: Optional[int] = None, linear_dtype=torch.bfloat16, attn_dtype=torch.bfloat16):
        """Random-init model materialised layer by layer on `device` (14B bf16 = 29.5 GB never
        exists twice): every decoder layer's q/k/v and gate/up matrices are fused as they are drawn, and with
        `linear_dtype=torch.float8_e4m3fn` quantised before the next layer is drawn; `attn_dtype` as in __init__."""
        from ..weights import global_weights, llm_layer_weights, vit_layer_weights

        check_linear_dtype(linear_dtype)
        check_attn_dtype(attn_dtype)
        w = global_weights(cfg, seed, device, torch.bfloat16, perturb)
        for i in range(cfg.visual.num_hidden_layers):
            w.update(vit_layer_weights(cfg, i, seed, device, torch.bfloat16, perturb))
        n_layers = cfg.num_hidden_layers if num_layers is None else num_layers
        layers = (DecoderLayer(cfg, llm_layer_weights(cfg, i, seed, device, torch.bfloat16, perturb), i, linear_dtype)
                  for i in range(n_layers))
        return cls(cfg, w, layers, linear_dtype, attn_dtype)

    def forward(
        self,
        input_ids: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        images: Optional[torch.Tensor] = None,
        image_indices: Optional[torch.Tensor] = None,
        position_ids: Optional[torch.Tensor] = None,
        past_key_values=None,
        inputs_embeds: Optional[torch.Tensor] = None,
        labels: Optional[torch.Tensor] = None,
        use_cache: Optional[bool] = None,
        output_attentions: Optional[bool] = None,
        output_hidden_states: Optional[bool] = None,
        return_dict: Optional[bool] = None,
        cache_position: Optional[torch.Tensor] = None,
        num_logits_to_keep: int = 0,
        **kwargs,
    ):
        outputs = self.model(
            input_ids=input_ids, attention_mask=attention_mask, images=images, image_indices=image_indices,
            position_ids=position_ids, past_key_values=past_key_values, inputs_embeds=inputs_embeds,
            use_cache=use_cache, output_attentions=output_attentions, output_hidden_states=output_hidden_states,
            return_dict=True, cache_position=cache_position, **kwargs,
        )
        hidden = outputs.last_hidden_state  # [1, s, H]
        # hidden_states[:, -num_logits_to_keep:, :] (modeling_long_vita.py:311); 0 keeps every row
        sel = hidden[:, -num_logits_to_keep:, :] if num_logits_to_keep else hidden
        rows = sel.reshape(-1, sel.shape[-1])
        logits = ops.linear(rows, self.lm_head).view(1, sel.shape[1], -1)
        loss = None
        if labels is not None:
            # transformers' loss_function (ForCausalLMLoss): labels shifted by one, mean of the per-token CE in fp32 over
            # the labels != -100.  Per-token CE from the chunked LM-head + CE kernels (ops.lm_head_ce_fwd): same bf16
            # logits, fp32 loss, and no fp32 copy of the [s, vocab] logits.
            tgt = labels[:, -logits.shape[1]:][:, 1:].reshape(-1).to(rows.device)
            per_tok, _ = ops.lm_head_ce_fwd(rows[:-1], self.lm_head, torch.where(tgt == -100, torch.full_like(tgt, -1), tgt))
            n_valid = (tgt != -100).sum().clamp_min(1)
            loss = per_tok.sum() / n_valid
        out = CausalLMOutput(loss=loss, logits=logits, past_key_values=outputs.past_key_values,
                             hidden_states=outputs.hidden_states)
        return out if (return_dict is None or return_dict) else out.to_tuple()

    @torch.no_grad()
    def prefill_context(self, input_ids: torch.Tensor, images: Optional[torch.Tensor] = None,
                        image_indices: Optional[torch.Tensor] = None, *,
                        kv_host_dtype=torch.bfloat16) -> ContextCache:
        """Prefill a prompt (a long video) once, for several questions about it: the prefill of
        `forward(use_cache=True, num_logits_to_keep=1, max_cache_len=s)` - the same placement of the cache, device or
        partly in pinned host memory (`kv_host_dtype` for its host tier), the same streaming and the same logits - with
        no spare rows, returned as a read-only kv_cache.ContextCache.  Ask with `generate(question, context=ctx)` or
        `forward(input_ids=question, past_key_values=ctx.session(n), use_cache=True)`."""
        dev = self.device
        s = input_ids.shape[1]
        if images is not None:
            images = images.to(dev, dtype=torch.bfloat16)
        if image_indices is not None:
            image_indices = image_indices.to(dev)
        out = self.forward(input_ids=input_ids.to(dev), images=images, image_indices=image_indices, use_cache=True,
                           num_logits_to_keep=1, max_cache_len=s, kv_host_dtype=kv_host_dtype)
        cfg = self.config
        return ContextCache(out.past_key_values, out.logits, cfg.num_key_value_heads, cfg.head_dim)

    @torch.no_grad()
    def generate(self, inputs: Optional[torch.Tensor] = None, images: Optional[torch.Tensor] = None,
                 image_indices: Optional[torch.Tensor] = None, generation_config=None, input_ids: Optional[torch.Tensor] = None,
                 max_new_tokens: Optional[int] = None, eos_token_id=None, do_sample: Optional[bool] = None,
                 kv_host_dtype=torch.bfloat16, context: Optional[ContextCache] = None, **kwargs):
        """`model.generate(inputs=, images=, image_indices=)` as tools/inference_long_vita.py:868 calls it: greedy
        decoding (the script sets do_sample = False) with the K/V cache; stops at `eos_token_id` (int or list) or after
        `max_new_tokens`; returns prompt + generated ids [1, s + n] like transformers' GenerationMixin.  Inputs on the
        host are moved to the model's device (the script leaves them on the CPU under device_map="auto").
        `kv_host_dtype=torch.float8_e4m3fn` keeps the host tier of a cache that does not fit in HBM in FP8 (lossy).

        With `context` (a ContextCache from prefill_context), `inputs` is a question about the context's prompt: it
        runs in a new session of the context (ContextCache.session), which the context outlives unchanged, and the
        result is question + answer ids.  The images belong to the context's prompt, so none are taken here."""
        if context is not None and images is not None:
            raise ValueError("generate(context=): the images belong to the context's prompt (prefill_context)")
        gc = generation_config if generation_config is not None else self.generation_config
        ids = inputs if inputs is not None else input_ids
        if ids is None:
            raise ValueError("generate() needs `inputs` (token ids [1, s])")
        sample = getattr(gc, "do_sample", False) if do_sample is None else do_sample
        if sample or kwargs.get("num_beams", 1) not in (None, 1):
            raise NotImplementedError("greedy decoding only (the reference's inference script: do_sample = False)")
        n_new = max_new_tokens if max_new_tokens is not None else (getattr(gc, "max_new_tokens", None) or 1024)
        eos = eos_token_id if eos_token_id is not None else getattr(gc, "eos_token_id", None)
        eos = set() if eos is None else ({int(eos)} if isinstance(eos, int) else {int(e) for e in eos})
        dev = self.device
        ids = ids.to(dev)
        if images is not None:
            images = images.to(dev, dtype=torch.bfloat16)
        if image_indices is not None:
            image_indices = image_indices.to(dev)
        cache = None if context is None else context.session(ids.shape[1] + int(n_new))
        new = self.generate_greedy(ids, images, image_indices, max_new_tokens=int(n_new), eos_token_ids=eos,
                                   kv_host_dtype=kv_host_dtype, cache=cache)
        return torch.cat([ids, new], dim=1)

    @torch.no_grad()
    def generate_greedy(self, input_ids: torch.Tensor, images: Optional[torch.Tensor] = None,
                        image_indices: Optional[torch.Tensor] = None, max_new_tokens: int = 16,
                        eos_token_id: Optional[int] = None, eos_token_ids=None,
                        kv_host_dtype=torch.bfloat16, cache=None) -> torch.Tensor:
        """Greedy decoding with the K/V cache: one prefill, then one forward per token over a single new
        row (the reference's Megatron loop feeds the whole sequence again for every token,
        generation.py:127-135).  With `cache` (a kv_cache.ContextSession) the prefill is that of the input rows
        after the cache's.  Returns the generated ids [1, n]."""
        s = input_ids.shape[1]
        stop = set(eos_token_ids or ())
        if eos_token_id is not None:
            stop.add(int(eos_token_id))
        if cache is None:
            out = self.forward(input_ids=input_ids, images=images, image_indices=image_indices, use_cache=True,
                               num_logits_to_keep=1, max_cache_len=s + max_new_tokens, kv_host_dtype=kv_host_dtype)
        else:
            out = self.forward(input_ids=input_ids, past_key_values=cache, use_cache=True, num_logits_to_keep=1)
        cache = out.past_key_values
        new = []
        tok = out.logits[0, -1].float().argmax().view(1, 1)
        for _ in range(max_new_tokens):
            new.append(tok)
            if stop and int(tok) in stop:
                break
            if len(new) == max_new_tokens:
                break
            out = self.forward(input_ids=tok, past_key_values=cache, use_cache=True, num_logits_to_keep=1)
            tok = out.logits[0, -1].float().argmax().view(1, 1)
        return torch.cat(new, dim=1)
