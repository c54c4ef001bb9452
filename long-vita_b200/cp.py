"""Context parallelism (zig-zag sequence sharding) - host side.

Layout contract (long_vita_megatron/training/utils.py:252-343, generation.py:517-566): the sequence
is cut into 2*cp chunks, rank r owns chunks {r, 2cp-1-r}; tokens, position ids and the RoPE table
are sliced the same way; an image is encoded by every rank that owns at least one of its tokens and
its features are scattered through (src_indices, tgt_indices).

The pure index logic (`zigzag_index`, `shard_prompt`) runs on any device and is covered by
world_size-2 gloo tests on CPU.  `CPContext` owns the peer-mapped K/V buffers (CUDA IPC through the
C ABI) and `ContextParallelRunner` runs the sharded prefill with the fused in-kernel K/V exchange
(`lv_attn_cp_fwd`) - no NCCL call sits on the attention path; NCCL only gathers the final logits.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


# ------------------------------------------------------------------------------------------------
# index logic (device-agnostic, bit-exact)
# ------------------------------------------------------------------------------------------------
def zigzag_index(seq_len: int, cp: int, rank: int, device=None) -> torch.Tensor:
    """Global positions owned by `rank`, in local order (chunk r then chunk 2cp-1-r)."""
    if seq_len % (2 * cp) != 0:
        raise ValueError(f"sequence length {seq_len} is not divisible by 2*cp = {2 * cp}")
    c = seq_len // (2 * cp)
    return torch.cat([torch.arange(rank * c, (rank + 1) * c, device=device),
                      torch.arange((2 * cp - 1 - rank) * c, (2 * cp - rank) * c, device=device)])


def zigzag_unpermute_index(seq_len: int, cp: int, device=None) -> torch.Tensor:
    """inv such that cat_r(local_r)[inv] is in global order (generation.py:548-564)."""
    order = torch.cat([zigzag_index(seq_len, cp, r, device) for r in range(cp)])
    inv = torch.empty_like(order)
    inv[order] = torch.arange(seq_len, device=device)
    return inv


@dataclass
class PromptShard:
    input_ids: torch.Tensor        # [1, 2c] local token ids
    position_ids: torch.Tensor     # [2c]    global positions of the local tokens
    image_sel: torch.Tensor        # [n_local_images] indices into the global image list
    src_idx: torch.Tensor          # flat indices into feat.view(-1, H) of the local images
    dst_idx: torch.Tensor          # matching local token rows
    last_token_local: int          # local row of the last global token, or -1


def shard_prompt(input_ids: torch.Tensor, image_indices: Optional[torch.Tensor], cp: int, rank: int,
                 tokens_per_image: int = 256) -> PromptShard:
    """get_batch_on_this_cp_rank for one sample (training/utils.py:252-343): slice tokens, keep the
    images with at least one token on this rank, translate global scatter targets to local rows."""
    b, S = input_ids.shape
    assert b == 1
    dev = input_ids.device
    own = zigzag_index(S, cp, rank, dev)
    local_of_global = torch.full((S,), -1, dtype=torch.int64, device=dev)
    local_of_global[own] = torch.arange(own.numel(), device=dev)
    ids_l = input_ids[:, own]
    if image_indices is not None and image_indices.numel() > 0:
        idx_s = image_indices[1]                       # [n_img, 256] global positions
        loc = local_of_global[idx_s]                   # -1 where the token lives on another rank
        mask = loc >= 0
        sel = mask.any(dim=1).nonzero().view(-1)
        m = mask[sel]
        n_sel = sel.numel()
        src_b = torch.arange(n_sel, device=dev).unsqueeze(1).expand(n_sel, idx_s.shape[1])
        src_s = torch.arange(idx_s.shape[1], device=dev).unsqueeze(0).expand(n_sel, idx_s.shape[1])
        src = (src_b * tokens_per_image + src_s)[m]
        dst = loc[sel][m]
    else:
        sel = torch.empty(0, dtype=torch.int64, device=dev)
        src = torch.empty(0, dtype=torch.int64, device=dev)
        dst = torch.empty(0, dtype=torch.int64, device=dev)
    last = int(local_of_global[S - 1])
    return PromptShard(ids_l, own, sel, src, dst, last)


# ------------------------------------------------------------------------------------------------
# peer-mapped buffers
# ------------------------------------------------------------------------------------------------
class _RawCudaBuffer:
    """Expose a raw device allocation to torch through __cuda_array_interface__ (int16 view)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes // 2,), "typestr": "<i2", "data": (ptr, False), "version": 3}


def _wrap_bf16(ptr: int, shape, device) -> torch.Tensor:
    n = math.prod(shape)
    t = torch.as_tensor(_RawCudaBuffer(ptr, n * 2), device=device)
    return t.view(torch.bfloat16).view(*shape)


class CPBackwardMixin:
    """Backward of the context-parallel attention (SURVEY.md 8a-2: "bwd ring for dKV"), first version:
    a composition of the single-GPU backward kernels with two collectives of the CP group.

      1. K/V of the whole sequence: all-gather of the ranks' local rows, re-ordered from zig-zag to
         global order (`lv_row_gather`, bit-exact);
      2. `lv_attn_bwd` on the local queries (two segments at their global positions) against the full
         K/V: dQ is final; dK/dV are this rank's partial sums over the kv rows its queries see (the
         kernel writes zeros for kv tiles no local query sees);
      3. partial dK|dV rows re-ordered to rank-major zig-zag order and reduce-scattered to their owners.

    The exchange volume per layer is 2 x S x hkv x d bf16 each way - under 1 % of the backward's run
    time at the lengths context parallelism is used for (128K, cp 8: ~1 ms vs ~150 ms), which is why
    this version uses the group's collectives instead of the forward's in-kernel pull.  Needs from the
    host class: group, cp, rank, S, T, hkv, d."""

    def _order(self, device):
        if getattr(self, "_order_cache", None) is None or self._order_cache[0].device != torch.device(device):
            order = torch.cat([zigzag_index(self.S, self.cp, r, device) for r in range(self.cp)])   # rank-major -> global pos
            self._order_cache = (order, zigzag_unpermute_index(self.S, self.cp, device))
        return self._order_cache

    def gather_kv(self, k: torch.Tensor, v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """k, v [T, hkv, d] local rows (zig-zag order) -> K, V [S, hkv, d] in global order."""
        from . import ops

        row = self.hkv * self.d
        local = torch.cat([k.reshape(self.T, row), v.reshape(self.T, row)], dim=1).contiguous()     # [T, 2 row]
        allr = torch.empty((self.cp * self.T, 2 * row), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(allr, local, group=self.group)
        full = ops.row_gather(allr, self._order(local.device)[1])                                    # global order
        return full[:, :row].view(self.S, self.hkv, self.d), full[:, row:].view(self.S, self.hkv, self.d)

    def reduce_dkv(self, dk_partial: torch.Tensor, dv_partial: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """partials [S, hkv, d] (global order) -> this rank's summed rows [T, hkv, d] (zig-zag order)."""
        from . import ops

        row = self.hkv * self.d
        part = torch.cat([dk_partial.reshape(self.S, row), dv_partial.reshape(self.S, row)], dim=1).contiguous()
        by_rank = ops.row_gather(part, self._order(part.device)[0])                                  # [cp * T, 2 row]
        mine = torch.empty((self.T, 2 * row), dtype=part.dtype, device=part.device)
        dist.reduce_scatter_tensor(mine, by_rank, group=self.group)
        return mine[:, :row].reshape(self.T, self.hkv, self.d), mine[:, row:].reshape(self.T, self.hkv, self.d)

    def attention_backward(self, d_out, q, k, v, out, lse, scale: Optional[float] = None):
        """d_out / q / out [T, hq, d], k / v [T, hkv, d] local rows, lse [1, hq, T] -> dq, dk, dv (local)."""
        from . import ops

        c = self.S // (2 * self.cp)
        K, V = self.gather_kv(k, v)
        dq, dk_p, dv_p = ops.attention_bwd(d_out.unsqueeze(0), q.unsqueeze(0), K.unsqueeze(0), V.unsqueeze(0),
                                           out.unsqueeze(0), lse, causal=True, scale=scale, q_seg_len=c,
                                           q_seg_pos=(self.rank * c, (2 * self.cp - 1 - self.rank) * c))
        dk, dv = self.reduce_dkv(dk_p[0], dv_p[0])
        return dq[0], dk, dv


def _refuse_packing(cu_seqlens) -> None:
    """Packed samples under context parallelism would need a document-aware exchange (the copier and the key walk of
    lv_attn_cp_fwd); the reference's own CP path for packed samples is not runnable either.  Refuse, never ignore."""
    if cu_seqlens is not None:
        raise NotImplementedError("packed samples (cu_seqlens / --reset-attention-mask) under context parallelism are "
                                  "not supported")


class _CPAttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, cp_ctx, scale):
        out, lse = cp_ctx.attention_separate(q, k, v, scale=scale, return_lse=True)
        T, hq, d = q.shape
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.cp_ctx, ctx.scale = cp_ctx, scale
        return out

    @staticmethod
    def backward(ctx, d_out):
        q, k, v, out, lse = ctx.saved_tensors
        T, hq, d = q.shape
        dq, dk, dv = ctx.cp_ctx.attention_backward(d_out.reshape(T, hq, d).contiguous(), q, k, v, out.view(T, hq, d), lse,
                                                   scale=ctx.scale)
        return dq, dk, dv, None, None


def cp_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cp_ctx, scale: Optional[float] = None,
                 cu_seqlens=None) -> torch.Tensor:
    """Differentiable context-parallel causal attention: q [T, hq, d], k / v [T, hkv, d] are this
    rank's zig-zag rows; returns [T, hq * d].  Forward = the fused in-kernel exchange
    (`lv_attn_cp_fwd`), backward = CPBackwardMixin.attention_backward.  Packed documents (`cu_seqlens`) raise."""
    _refuse_packing(cu_seqlens)
    return _CPAttentionFn.apply(q, k, v, cp_ctx, scale)


class CPContext(CPBackwardMixin):
    """Per-process context-parallel state: two peer-mapped QKV buffers (epoch parity), the ready
    words, the local K/V staging buffers and block flags; peers' mappings opened via CUDA IPC."""

    _shared = {}
    MAX_SHARED = 2     # geometries kept alive per process (e.g. the training and the evaluation sequence length)

    @classmethod
    def shared(cls, group, seq_total, hq, hkv, d, device, fused_qkv=True):
        """One context per (group, geometry): all layers of a model share the buffers and the epoch.  The cache is
        bounded: a geometry beyond MAX_SHARED evicts (and closes) the least recently used one, so prompts of varying
        length do not pile up peer-mapped allocations (every rank makes the same calls in the same order, so every rank
        evicts the same context - `close()` is collective)."""
        key = (id(group), seq_total, hq, hkv, d, str(device), fused_qkv)
        ctx = cls._shared.pop(key, None)
        if ctx is None:
            while len(cls._shared) >= cls.MAX_SHARED:
                cls._shared.pop(next(iter(cls._shared))).close()
            ctx = cls(group, seq_total, hq, hkv, d, device, fused_qkv)
        cls._shared[key] = ctx          # most recently used last
        return ctx

    def __init__(self, group, seq_total: int, hq: int, hkv: int, d: int, device, fused_qkv: bool = True):
        from . import _lib

        self.lib = _lib.lib()
        self._check = _lib.check
        self.group = group
        self.cp = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        if not (2 <= self.cp <= 8):
            raise ValueError("context-parallel size must be in [2, 8] (one NVSwitch node)")
        self.S, self.hq, self.hkv, self.d = seq_total, hq, hkv, d
        self.device = device
        self.T = seq_total // self.cp
        self.fused_qkv = fused_qkv
        # peer-mapped rows hold either the whole fused QKV GEMM output (zero-copy path) or K|V only
        self.row = (hq + 2 * hkv) * d if fused_qkv else 2 * hkv * d
        self.k_col = hq * d if fused_qkv else 0
        self.epoch = 0
        qkv_bytes = self.T * self.row * 2
        self.flag_bytes = 256
        total = 2 * qkv_bytes + self.flag_bytes
        base = C.c_void_p()
        self._check(self.lib.lv_ipc_alloc(total, C.byref(base)), "lv_ipc_alloc")
        self.base = base.value
        self.qkv = [_wrap_bf16(self.base + i * qkv_bytes, (self.T, self.row), device) for i in range(2)]
        self.ready_ptr = self.base + 2 * qkv_bytes
        # exchange IPC handles
        h = (C.c_ubyte * 64)()
        self._check(self.lib.lv_ipc_get_handle(self.base, h), "lv_ipc_get_handle")
        mine = torch.tensor(list(h), dtype=torch.uint8, device=device)
        allh = [torch.empty_like(mine) for _ in range(self.cp)]
        dist.all_gather(allh, mine, group=group)
        self.peer_base: List[int] = []
        for p in range(self.cp):
            if p == self.rank:
                self.peer_base.append(self.base)
                continue
            hb = (C.c_ubyte * 64)(*allh[p].cpu().tolist())
            pp = C.c_void_p()
            self._check(self.lib.lv_ipc_open_handle(hb, C.byref(pp)), "lv_ipc_open_handle")
            self.peer_base.append(pp.value)
        self.qkv_bytes = qkv_bytes
        self.k_full = torch.empty((seq_total, hkv * d), dtype=torch.bfloat16, device=device)
        self.v_full = torch.empty((seq_total, hkv * d), dtype=torch.bfloat16, device=device)
        self.blk_flags = torch.zeros(seq_total // 128, dtype=torch.int32, device=device)
        self.fault = torch.zeros(1, dtype=torch.int32, device=device)     # sticky: set by a kernel whose peer wait timed out
        dist.barrier(group=group)

    def close(self) -> None:
        """Collective over the group: unmap the peers' buffers and free this rank's.  An exporter's allocation stays
        pinned while any peer still maps it, so the order is: everyone's kernels done -> everyone closes its
        mappings -> everyone frees.  Idempotent."""
        if self.base is None:
            return
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)
        self.qkv = []
        for p, ptr in enumerate(self.peer_base):
            if p != self.rank:
                self._check(self.lib.lv_ipc_close_handle(ptr), "lv_ipc_close_handle")
        self.peer_base = []
        dist.barrier(group=self.group)
        self._check(self.lib.lv_ipc_free(self.base), "lv_ipc_free")
        self.base = None
        self.k_full = self.v_full = self.blk_flags = self.fault = None

    def check(self) -> None:
        """Raise (LV_ESTATE) if any attention kernel of this context gave up waiting for a peer rank: every in-kernel
        wait on another GPU is bounded (LV_CP_TIMEOUT_MS), so a dead or diverged peer costs an error here instead of a
        hung node.  Synchronises the current stream - call it where the host reads a result anyway."""
        if self.base is None:      # closed
            return
        self._check(self.lib.lv_cp_check_fault(self.fault.data_ptr(), torch.cuda.current_stream().cuda_stream), "lv_cp_check_fault")

    def qkv_buffer(self) -> torch.Tensor:
        """The peer-mapped [T, row] buffer the NEXT attention call reads: the fused QKV GEMM writes
        it directly (fused_qkv) or attention_separate() copies K|V into it."""
        return self.qkv[self.epoch & 1]

    def attention(self, out: Optional[torch.Tensor] = None, scale: Optional[float] = None,
                  lse: Optional[torch.Tensor] = None, cu_seqlens=None) -> torch.Tensor:
        """Causal attention of the local queries (already RoPE'd, inside qkv_buffer()) over the whole
        sequence; K/V of the other ranks are pulled by the kernel.  Returns [T, hq*d]; `lse` ([1, hq, T] fp32,
        optional) receives the log-sum-exp.  Packed documents (`cu_seqlens`) raise NotImplementedError."""
        _refuse_packing(cu_seqlens)
        assert self.fused_qkv
        q = self.qkv[self.epoch & 1][:, : self.hq * self.d].view(self.T, self.hq, self.d)
        return self._launch(q, out, scale, lse)

    def attention_separate(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out=None, scale=None,
                           return_lse: bool = False, cu_seqlens=None):
        """q [T, hq, d], k/v [T, hkv, d] (strided views are fine): K|V are copied into the peer-mapped
        buffer (T * 2 hkv d elements - small next to the attention itself), Q is read in place.
        With return_lse also returns the log-sum-exp [1, hq, T] fp32 (what the backward needs).  Packed documents
        (`cu_seqlens`) raise NotImplementedError."""
        _refuse_packing(cu_seqlens)
        assert not self.fused_qkv
        buf = self.qkv[self.epoch & 1].view(self.T, 2, self.hkv, self.d)
        buf[:, 0].copy_(k)
        buf[:, 1].copy_(v)
        from . import ops

        lse = torch.empty((1, self.hq, self.T), dtype=torch.float32, device=self.device) if return_lse else None
        o = self._launch(ops.tma_view(q), out, scale, lse)
        return (o, lse) if return_lse else o

    def _launch(self, q, out, scale, lse=None):
        """q [T, hq, d]: this rank's queries, read in place.  K/V are the global-order staging buffers the kernel fills."""
        from . import ops
        from ._lib import CpParams

        T, hq, hkv, d = self.T, self.hq, self.hkv, self.d
        par = self.epoch & 1
        if out is None:
            out = torch.empty((T, hq * d), dtype=torch.bfloat16, device=self.device)
        c = self.S // (2 * self.cp)
        a = ops.attn_params(q.unsqueeze(0), self.k_full.view(1, self.S, hkv, d), self.v_full.view(1, self.S, hkv, d),
                            out.view(1, T, hq, d), lse, scale=scale, causal=True, q_seg_len=c,
                            q_seg_pos=(self.rank * c, (2 * self.cp - 1 - self.rank) * c))
        cpp = CpParams()
        cpp.rank, cpp.cp, cpp.seq_total, cpp.epoch = self.rank, self.cp, self.S, self.epoch
        cpp.peer_tok_stride = self.row
        k_off = (par * self.qkv_bytes) + self.k_col * 2
        for p in range(self.cp):
            cpp.peer_kv[p] = self.peer_base[p] + k_off
            cpp.peer_ready[p] = self.peer_base[p] + 2 * self.qkv_bytes
        cpp.my_ready = self.ready_ptr
        cpp.k_full, cpp.v_full, cpp.blk_flags = self.k_full.data_ptr(), self.v_full.data_ptr(), self.blk_flags.data_ptr()
        cpp.fault = self.fault.data_ptr()
        ev0 = ops._TIMER.start() if ops._TIMER is not None else None
        self._check(self.lib.lv_attn_cp_fwd(C.byref(a), C.byref(cpp), torch.cuda.current_stream().cuda_stream),
                    "lv_attn_cp_fwd")
        if ev0 is not None:
            ops._TIMER.stop("attn_fwd", 4.0 * hq * d * (self.S * (self.S + 1) / 2) / self.cp, ev0)
        self.epoch += 1
        return out


# ------------------------------------------------------------------------------------------------
# sharded prefill
# ------------------------------------------------------------------------------------------------
def exchange_attention(ctx, cache=None):
    """Attention step (hf.modeling.run_layers) of a decoder layer on this rank's zig-zag shard: the QKV GEMM wrote
    into `ctx.qkv_buffer()` and RoPE ran in place there; the fused kernel pulls the other ranks' K/V itself
    (lv_attn_cp_fwd).  With `cache`, this rank's rows become its shard of the K/V cache."""
    def attend(li, q, k, v):
        if cache is not None:
            cache.append(li, k, v)
        return ctx.attention()

    return attend


class ContextParallelRunner:
    """LongVITAForCausalLM prefill with the sequence sharded zig-zag over the ranks of `group`."""

    def __init__(self, model, group):
        self.model = model
        self.group = group
        self.cp = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.ctx: Optional[CPContext] = None
        self.check_faults = True   # synchronise + read the exchange's fault word at the end of every forward
        self.cache = None          # this rank's K/V cache shard after forward(..., use_cache=True)
        self.total_len = 0         # tokens in the whole (sharded) cache

    def _context(self, S: int, device) -> CPContext:
        cfg = self.model.config
        if self.ctx is None or self.ctx.S != S:
            if self.ctx is not None:
                self.ctx.close()       # a new prompt length: release the peer-mapped buffers of the old one first
            self.ctx = CPContext(self.group, S, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim, device)
        return self.ctx

    def close(self) -> None:
        if self.ctx is not None:
            self.ctx.close()
            self.ctx = None

    def forward(self, input_ids: torch.Tensor, images: Optional[torch.Tensor], image_indices: Optional[torch.Tensor],
                gather_logits: bool = True, use_cache: bool = False, max_new_tokens: int = 1024) -> torch.Tensor:
        """Every rank passes the FULL prompt (the reference broadcasts it, tasks/inference/module.py
        :340-356) and keeps its shard.  Returns the last-token logits [1, 1, vocab] on every rank."""
        from . import ops
        from .hf.modeling import run_layers

        m = self.model.model
        cfg = self.model.config
        dev = input_ids.device
        S = input_ids.shape[1]
        ctx = self._context(S, dev)
        sh = shard_prompt(input_ids, image_indices, self.cp, self.rank, cfg.visual.tokens_per_image)
        feat = None
        if images is not None and sh.image_sel.numel() > 0:
            feat = m.encode_images(images[sh.image_sel])
        x = ops.embed_scatter(sh.input_ids, m.embed_tokens, feat, sh.dst_idx if feat is not None else None,
                              sh.src_idx if feat is not None else None)
        feat = None                         # scattered into x: not held through the decoder
        cos, sin = ops.rope_table(sh.position_ids.to(torch.int64), m.inv_freq)
        T = x.shape[0]
        self.cache = None
        if use_cache:      # this rank's shard of the K/V cache: its T zig-zag rows + its share of the new tokens
            from .kv_cache import KVCache

            self.cache = KVCache(len(m.layers), T + -(-max_new_tokens // self.cp) + 1, cfg.num_key_value_heads, cfg.head_dim, dev)
            self.total_len = S
        h = run_layers(m.layers, x, cos, sin, exchange_attention(ctx, self.cache), m.norm_w, cfg.rms_norm_eps,
                       cache=self.cache, qkv_out=ctx.qkv_buffer, donate=True)
        # logit mask: each rank projects its own last row; the globally-last token lives on rank 0
        # (chunk 2cp-1), generation.py:141-165
        row = sh.last_token_local if sh.last_token_local >= 0 else T - 1
        logits = ops.linear(h[row : row + 1], self.model.lm_head).view(1, 1, -1)
        if gather_logits:
            dist.broadcast(logits, src=dist.get_global_rank(self.group, 0), group=self.group)
        if self.check_faults:
            ctx.check()        # a peer that never published its K/V shows up here as an error, not as a hang
        return logits

    # -- incremental decoding over the sharded cache (SURVEY.md 8f-2 under context parallelism) --------------
    def _merge(self, o_loc: torch.Tensor, lse_loc: torch.Tensor) -> torch.Tensor:
        """Combine the ranks' partial attention results over their cache shards: out = sum_r w_r o_r with
        w_r = exp(lse_r - logsumexp_r lse_r).  One all-gather of [hq, d + 1] floats (20 KB at 40 x 128)."""
        hq, d = o_loc.shape
        pack = torch.cat([o_loc.float(), lse_loc.view(hq, 1)], dim=1).contiguous()
        allp = torch.empty((self.cp * hq, d + 1), dtype=torch.float32, device=pack.device)
        dist.all_gather_into_tensor(allp, pack, group=self.group)
        allp = allp.view(self.cp, hq, d + 1)
        w = torch.softmax(allp[:, :, d], dim=0)                   # -inf (empty shard) -> weight 0
        return (allp[:, :, :d] * w.unsqueeze(-1)).sum(dim=0).to(torch.bfloat16)

    def _shard_attention(self, append: bool):
        """Attention step of one decoded token over the sharded cache (any split of the keys works for a query that
        sees them all): this rank attends over its shard, `_merge` combines the ranks' (out, lse) pairs.  Only the rank
        that owns the new position (`append`) adds its K/V row."""
        from . import ops

        cache = self.cache

        def attend(li, q, k, v):
            if append:
                kc, vc, length = cache.append(li, k, v)
            else:
                kc, vc, length = cache.k[li], cache.v[li], len(cache)
            if length > 0:
                o_loc, lse_loc = ops.attention_decode(q[0], kc, vc, length, return_lse=True)
            else:
                hq, d = q.shape[1], q.shape[2]
                o_loc = torch.zeros((hq, d), dtype=torch.bfloat16, device=q.device)
                lse_loc = torch.full((hq,), float("-inf"), dtype=torch.float32, device=q.device)
            return self._merge(o_loc, lse_loc)

        return attend

    def decode(self, token: torch.Tensor) -> torch.Tensor:
        """One generated token after forward(..., use_cache=True): every rank runs the token through the
        (replicated) weights; attention reads only this rank's cache shard and the partial results are merged.
        The new K/V row goes to rank `position % cp`.  Returns the logits [1, 1, vocab] (same on every rank)."""
        from . import ops
        from .hf.modeling import run_layers

        m = self.model.model
        cfg = self.model.config
        assert self.cache is not None, "call forward(..., use_cache=True) first"
        pos = self.total_len
        x = ops.embed_scatter(token.view(1, 1), m.embed_tokens)
        cos, sin = ops.rope_table(torch.tensor([pos], dtype=torch.int64, device=x.device), m.inv_freq)
        h = run_layers(m.layers, x, cos, sin, self._shard_attention((pos % self.cp) == self.rank), m.norm_w,
                       cfg.rms_norm_eps, cache=self.cache)
        self.total_len += 1
        return ops.linear(h, self.model.lm_head).view(1, 1, -1)
