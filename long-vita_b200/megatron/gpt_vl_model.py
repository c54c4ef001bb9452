"""`GPTVLModel.forward` on the H100 kernels (SURVEY.md 8a-15) - Megatron-free.

Mirrors long_vita_megatron/core/models/multimodal/gpt_vl_model.py:233-416: same argument list, same
`external_inputs` conventions, same embedding merge modes
(long_vita_megatron/core/models/common/embeddings/language_model_embedding.py:102-134), the
logit-masked output layer (core/tensor_parallel/layers.py:402-409) and the `[s b h] -> [b s h]`
return (:379).  The state dict is the Megatron-core (TE-spec) one - see `checkpoint.mcore_to_hf`.

What is kept from the reference and what is deliberately not:
* `inference_params.external_inputs` / `.logit_mask` overrides (:268-272, :287-289) and
  `use_kv_cache == False -> inference_params = None` (:291-292) are honoured.  With a live `inference_params`
  (Megatron's `--use-kv-cache` protocol, generation.py:127-131: only the new tokens are passed) the K/V rows go
  to a pre-allocated `kv_cache.KVCache` kept in `inference_params.key_value_memory_dict` and a single new token
  runs the flash-decoding path.  A cache that does not fit in HBM is partly in pinned host memory
  (`hf.modeling.new_cache`, `kv_cache.OffloadedKVCache`).
* `hidden_states += 0.0 * self.unused` (:310-311) is an exact no-op on finite values and only exists
  to keep an otherwise unused parameter in the autograd graph; not executed.
* labels: `masked_select(labels, logit_mask)` (:389-391), the `is_instruction_dataset` shift
  (:396-398), the NaN check (:400-403, raises ValueError) and a per-token fp32 cross-entropy
  returned as [b, s'] (LanguageModule.compute_language_model_loss).  The loss is host-side torch on
  the [M, vocab] logits the masked head produced - off the hot path.
* micro-batch 1 (the reference's long-context setting; `assert b == 1` at :325, :385).

Packed samples (`--reset-position-ids --reset-attention-mask`): position ids that restart at 0 inside the row mark
sample boundaries (compute_actual_seq_len, training/utils.py:53-57); attention is then causal within each sample and
blind across samples (ops.packed_cu_seqlens -> lv_attn_docs_fwd), as the reference's flash-attention path does.  The
boundaries are read once per forward.  Packing is not combined with context parallelism or a KV cache (both raise).

Under context parallelism the caller passes this rank's shard exactly as
`get_batch_on_this_cp_rank` (training/utils.py:252-343) produces it: zig-zag `input_ids`,
`position_ids`, `logit_mask`, and `external_inputs = {images, src_indices, tgt_indices}`; pass the
rank's `CPContext` as `cp=`.
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch

from .. import kv_cache, ops
from ..config import LongVITAConfig
from ..cp import exchange_attention
from ..hf import modeling
from ..hf.modeling import (VISION_CHUNK, DecoderLayer, attention_step, encode_images, packed_rows, rope_inv_freq,
                           run_layers, vision_tower)
from .checkpoint import mcore_to_hf


class B200GPTVLModel:
    def __init__(self, cfg: LongVITAConfig, state_dict: Dict[str, torch.Tensor], *, pre_process: bool = True,
                 post_process: bool = True, cp=None, is_instruction_dataset: bool = False,
                 output_multiplier_scale: Optional[float] = None, output_logit_softcapping: Optional[float] = None,
                 gradient_accumulation_fusion: bool = False, kv_host_dtype=torch.bfloat16):
        if not (pre_process and post_process):
            raise NotImplementedError("pipeline parallelism is not built (14B bf16 fits one 80 GB H100: pp = 1)")
        self.config = cfg
        self.pre_process, self.post_process = pre_process, post_process
        self.cp = cp
        self.is_instruction_dataset = is_instruction_dataset
        self.output_multiplier_scale = output_multiplier_scale
        self.output_logit_softcapping = output_logit_softcapping
        # Megatron's config.gradient_accumulation_fusion for the output layer: when output_weight requires grad, its
        # gradient is added to output_weight.main_grad (fp32) inside the GEMM (ops.masked_lm_head_ce / masked_linear)
        self.gradient_accumulation_fusion = bool(gradient_accumulation_fusion)
        # the format of the host tier of a K/V cache the inference_params path creates (kv_cache.make_cache): bf16, or
        # the lossy FP8 e4m3 one that halves its pinned memory and decode traffic
        self.kv_host_dtype = kv_cache.check_host_dtype(kv_host_dtype)
        w = mcore_to_hf(state_dict, cfg)
        self.word_embeddings = w["model.embed_tokens.weight"]
        self.final_layernorm = w["model.norm.weight"]
        self.output_weight = w["lm_head.weight"]
        self.layers = [DecoderLayer(cfg, w, i) for i in range(cfg.num_hidden_layers)
                       if f"model.layers.{i}.self_attn.q_proj.weight" in w]
        self.vit, self.vision_projection = vision_tower(cfg, w)
        self.inv_freq = rope_inv_freq(cfg, self.word_embeddings.device)
        self.vision_chunk = VISION_CHUNK

    # -- external_feature_model(**external_inputs) (pretrain_long_vita.py:535-563) -----------------
    def external_feature_model(self, images: torch.Tensor, **_unused) -> torch.Tensor:
        return encode_images(self.vit, self.vision_projection, images, self.vision_chunk)

    @staticmethod
    def _indices_dst(indices: torch.Tensor, s: int, dev) -> torch.Tensor:
        """The flat rows of `indices` mode ([2, n, tokens]: batch, position) in a row of s tokens."""
        idx_b, idx_s = indices.to(dev).unbind(dim=0)
        return (idx_b.reshape(-1) * s + idx_s.reshape(-1)).to(torch.int64)

    # -- LanguageModelEmbedding.forward (language_model_embedding.py:91-134) -> [s, h] --------------
    def embedding(self, input_ids: torch.Tensor, position_ids, external_feature_dict: Optional[dict] = None):
        b, s = input_ids.shape
        if b != 1:
            raise NotImplementedError("micro-batch 1 (the reference's long-context setting)")
        if external_feature_dict is None:
            return ops.embed_scatter(input_ids, self.word_embeddings)
        d = external_feature_dict
        ok = "features" in d and (
            len(d) == 1 or (len(d) == 2 and "pre_len" in d) or (len(d) == 2 and "indices" in d)
            or (len(d) == 3 and "src_indices" in d and "tgt_indices" in d))
        assert ok, "The format of external_feature_dict is not right!"
        feat = d["features"]
        dev = input_ids.device
        if "indices" in d:
            return ops.embed_scatter(input_ids, self.word_embeddings, feat, self._indices_dst(d["indices"], s, dev))
        if "pre_len" in d:
            if feat.shape[0] != 1:
                raise NotImplementedError("pre_len mode broadcasts one feature block per batch row; batch is 1")
            dst = int(d["pre_len"]) + torch.arange(feat.shape[1], device=dev, dtype=torch.int64)
            return ops.embed_scatter(input_ids, self.word_embeddings, feat, dst)
        if "src_indices" in d:
            src_b, src_s = d["src_indices"]
            tgt_b, tgt_s = d["tgt_indices"]
            src = (src_b.to(dev).reshape(-1) * feat.shape[1] + src_s.to(dev).reshape(-1)).to(torch.int64)
            dst = (tgt_b.to(dev).reshape(-1) * s + tgt_s.to(dev).reshape(-1)).to(torch.int64)
            if dst.numel() == 0:
                return ops.embed_scatter(input_ids, self.word_embeddings)
            return ops.embed_scatter(input_ids, self.word_embeddings, feat, dst, src)
        return ops.embed_scatter(input_ids, self.word_embeddings)     # features only: `+= features.mean() * 0`

    def forward(
        self,
        input_ids: torch.Tensor,
        position_ids: torch.Tensor,
        attention_mask: torch.Tensor,
        decoder_input: torch.Tensor = None,
        labels: torch.Tensor = None,
        inference_params=None,
        packed_seq_params=None,
        extra_block_kwargs: dict = None,
        external_inputs: dict = {},
        tokentype_ids=None,
        logit_mask=None,
    ) -> torch.Tensor:
        cfg = self.config
        assert packed_seq_params is None, "Packed sequence is not supported by flash attention."
        assert tokentype_ids is None
        if extra_block_kwargs:
            raise NotImplementedError(f"extra_block_kwargs {sorted(extra_block_kwargs)} are not supported")
        if decoder_input is not None:
            s, b, _ = decoder_input.shape
        else:
            b, s = input_ids.shape
            if (getattr(inference_params, "external_inputs", None) is not None
                    and not getattr(inference_params, "key_value_memory_dict", None)):
                external_inputs = inference_params.external_inputs
        if b != 1:
            raise NotImplementedError("micro-batch 1 (the reference's long-context setting)")
        if getattr(inference_params, "logit_mask", None) is not None:
            logit_mask = inference_params.logit_mask
        if hasattr(inference_params, "use_kv_cache") and not inference_params.use_kv_cache:
            inference_params = None
        dev = self.word_embeddings.device if decoder_input is None else decoder_input.device
        # Megatron's incremental decoding protocol (`--use-kv-cache`, generation.py:127-131): the caller passes only
        # the new tokens and their positions; per-layer K/V live in `inference_params.key_value_memory_dict`.  Here
        # that dict holds one pre-allocated cache for the whole model (hf.modeling.new_cache).
        cache = None
        if inference_params is not None:
            if self.cp is not None:
                raise NotImplementedError("KV-cache decoding under context parallelism goes through "
                                          "cp.ContextParallelRunner (sharded cache)")
            kv = inference_params.key_value_memory_dict
            cache = kv.get("b200_kv_cache")
            if cache is None:
                capacity = int(getattr(inference_params, "max_sequence_length", 0) or (s + 1024))
                cache = modeling.new_cache(cfg, len(self.layers), capacity, s, dev, self.kv_host_dtype)
                kv["b200_kv_cache"] = cache

        # RoPE: Megatron builds the table for positions 0..S-1 and slices it zig-zag under CP
        # (rotary_pos_embedding.py:36-47, 84-122); position_ids from get_batch_on_this_cp_rank are
        # exactly those positions, so the table is generated from them directly.
        cu = None
        if position_ids is None:
            assert self.cp is None, "context parallelism needs this rank's position_ids"
            p0 = 0 if cache is None else len(cache)
            position_ids = torch.arange(p0, p0 + s, device=dev).unsqueeze(0)
        else:
            cu = packed_rows(position_ids, s, dev, cache=cache, cp=self.cp)
        attend = attention_step(cache, cu, s) if self.cp is None else exchange_attention(self.cp)

        if decoder_input is not None:
            x = decoder_input.reshape(s, -1).contiguous()
        else:
            external_inputs = external_inputs or {}
            modes = [key for key in external_inputs if "indices" in key or key == "pre_len"]
            if modes == ["indices"] and modeling.streams(s, attend):
                # the decoder streams (hf.modeling.STREAM_THRESHOLD): so does the vision phase, each ViT chunk's
                # features going into x as soon as they are made
                x = self.embedding(input_ids, position_ids)
                dst = self._indices_dst(external_inputs["indices"], s, dev)
                x = modeling.scatter_images(x, self.vit, self.vision_projection, external_inputs["images"], dst,
                                            self.vision_chunk)
            elif external_inputs:
                feat = self.external_feature_model(**external_inputs)
                efd = {"features": feat}
                for key in external_inputs:
                    if "indices" in key or key == "pre_len":
                        efd[key] = external_inputs[key]
                x = self.embedding(input_ids, position_ids, efd)
                feat = efd = None                   # scattered into x: not held through the decoder
            else:
                x = self.embedding(input_ids, position_ids)
        cos, sin = ops.rope_table(position_ids.reshape(-1).to(torch.int64), self.inv_freq)

        h = run_layers(self.layers, x, cos, sin, attend, self.final_layernorm, cfg.rms_norm_eps, cache=cache,
                       qkv_out=None if self.cp is None else self.cp.qkv_buffer, donate=decoder_input is None)
        hidden_states = h.view(s, 1, -1)

        # training tail, fused: masked row gather -> LM head -> per-token cross-entropy, chunked over the vocabulary so
        # the [M, vocab] logits never exist (SURVEY.md 8f-3).  Taken when nothing between the head and the loss needs
        # the logits themselves (no multiplier / soft-capping; the NaN probe of :393 reads the loss instead).
        if (labels is not None and logit_mask is not None and not self.output_multiplier_scale
                and not self.output_logit_softcapping and getattr(self, "fused_loss", True)):
            assert logit_mask.size(0) == 1
            mask = logit_mask.to(hidden_states.device).to(torch.bool)
            with torch.no_grad():
                lab = torch.masked_select(labels.to(hidden_states.device), mask).reshape(1, -1)
            if self.is_instruction_dataset:
                # labels[:, 1:] against logits[:-1] (:386-388): drop the last selected row and the first label
                keep = mask.clone()
                last = mask.reshape(-1).nonzero().view(-1)[-1:]
                keep.view(-1)[last] = False
                mask, lab = keep, lab[:, 1:].contiguous()
            loss = ops.masked_lm_head_ce(hidden_states, self.output_weight, mask, lab,
                                         accumulate_wgrad=self.gradient_accumulation_fusion)
            if loss.sum().isnan():
                rank = torch.distributed.get_rank() if torch.distributed.is_initialized() else 0
                raise ValueError(f"Rank {rank}: found NaN in local forward logits calculation. "
                                 f"Device: {loss.device}, node: {os.uname()[1]}")
            return loss

        # output layer (ColumnParallelLinear with logit_mask, layers.py:402-409, 825-904)
        if logit_mask is not None:
            logits = ops.masked_linear(hidden_states, self.output_weight, logit_mask.to(hidden_states.device),
                                       accumulate_wgrad=self.gradient_accumulation_fusion)
        else:
            logits = ops.linear(hidden_states.view(s, -1), self.output_weight).view(s, 1, -1)
        if self.output_multiplier_scale:
            logits = logits * self.output_multiplier_scale
        if self.output_logit_softcapping:
            logits = torch.tanh(logits / self.output_logit_softcapping) * self.output_logit_softcapping
        if labels is None:
            return logits.transpose(0, 1).contiguous()              # [s b h] => [b s h]

        if logit_mask is not None:
            assert logit_mask.size(0) == 1
            with torch.no_grad():
                labels = torch.masked_select(labels, logit_mask.to(torch.bool)).reshape(1, -1)
        if self.is_instruction_dataset:
            labels = labels[:, 1:].contiguous()
            logits = logits[:-1, :, :].contiguous()
        if logits.sum().isnan():
            rank = torch.distributed.get_rank() if torch.distributed.is_initialized() else 0
            raise ValueError(f"Rank {rank}: found NaN in local forward logits calculation. "
                             f"Device: {logits.device}, node: {os.uname()[1]}")
        # compute_language_model_loss: per-token CE in fp32, [s b] -> [b s]
        lg = logits.float().reshape(-1, logits.shape[-1])
        loss = torch.nn.functional.cross_entropy(lg, labels.reshape(-1).to(lg.device), reduction="none")
        return loss.view(1, -1)

    __call__ = forward
